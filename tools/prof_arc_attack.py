"""Launch times of the ARC-aware attacks (rcmarl_pipeline_arc_attack, rcmarl_history_arc_attack) and the C2 round time
on arc_std against gauss, with every cooperative agent clipping (clipping="arc") before clip at H = 1:
  C2     5 agents, agent 4 on arc_std (s = 2): 3 receivers x 2 nets = 6 jobs per launch, n_in 4, P 661 / 761; the
         pipeline form against receivers without momentum, the history form against receivers on momentum 0.9
         (torch.profiler, CUDA activities: mean device time per launch over the profiled rounds, beside the base form
         of the same run with history_std)
  X32    32 jobs of 16 slots (15 real, 1 crafted), P 1421, clip at H = 1 (k_clip = 1): each form and its base form,
         CUDA events around `reps` launches after a warm-up
  round  one C2 update round (two epochs, the benchmark's hyper-parameters) on arc_std and on gauss, alternated,
         `rounds` times each: medians of the host clock around a round that ends in a device synchronise
The card's name and power limit are printed beside the numbers.

    python tools/prof_arc_attack.py [rounds=5] [out_dir]   -> prints one line per measurement (and a JSON file)
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "resilient-consensus-based-marl_b200"))
import bench                                   # noqa: E402
from rcmarl import ops                         # noqa: E402
from rcmarl.trainer import Trainer             # noqa: E402

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
out_dir = sys.argv[2] if len(sys.argv) > 2 else None


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def c2(attack, momentum=None):
    return Trainer(**dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=attack,
                          aggregation="clip", clipping="arc", momentum=momentum))


def kernel_us(prof, name):
    ev = [e for e in prof.events() if name in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    return (float(np.mean([e.device_time_total for e in ev])), len(ev)) if ev else (None, 0)


def c2_launches():
    rows = []
    for momentum, kernel in ((None, "pipeline_attack_kernel"), (0.9, "history_attack_kernel")):
        for name in ("arc_std", "history_std"):
            attack = (name, 2.0)
            clip = "arc" if name == "arc_std" else None
            tr = Trainer(**dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=attack,
                                aggregation="clip", clipping=clip, momentum=momentum))
            tr.rollout_block()
            tr.update_round()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(2):
                    tr.rollout_block()
                    tr.update_round()
                torch.cuda.synchronize()
            us, n = kernel_us(prof, kernel)
            rows.append(dict(shape="C2", momentum=momentum, attack=name, kernel=kernel, jobs=6, launches=n,
                             us_per_launch=us))
            print(f"C2  m{momentum} {name:11s} {kernel}: {us:9.1f} us per launch ({n} launches, 6 jobs)", flush=True)
    return rows


def x32(reps=20):
    rs = np.random.RandomState(3)
    P, S = 1421, 1427
    msgs = torch.as_tensor((rs.randn(1, S) + rs.randn(16, S) * 0.5).astype(np.float32)).cuda()
    ref = torch.as_tensor(rs.randn(S).astype(np.float32)).cuda()
    M = torch.as_tensor((rs.randn(16, S) * 0.3).astype(np.float32)).cuda()
    dst = torch.zeros(32, S, device="cuda")
    gam = torch.zeros(32, 1, device="cuda")
    slots = list(range(15)) + [-1]
    honest = list(range(15))
    jobs = {
        "pipeline_attack": (ops.pipeline_attack, [ops.pipeline_attack_job(dst[j], msgs, S, P, slots, honest, "clip", 1,
                                                                          "pipeline_std", 2.0, gamma_out=gam[j])
                                                  for j in range(32)]),
        "history_attack": (ops.history_attack, [ops.history_attack_job(dst[j], msgs, S, P, slots, honest, "clip", 1,
                                                                       "history_std", 2.0, ref, M, S, 0.9, 0, [15],
                                                                       gamma_out=gam[j]) for j in range(32)]),
    }
    jobs["pipeline_arc_attack"] = (ops.pipeline_arc_attack, jobs["pipeline_attack"][1])
    jobs["history_arc_attack"] = (ops.history_arc_attack, jobs["history_attack"][1])
    rows = []
    for name, (fn, js) in jobs.items():
        arr = ops.job_array(type(js[0]), js)
        fn(arr)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn(arr)
        b.record()
        torch.cuda.synchronize()
        us = a.elapsed_time(b) * 1e3 / reps
        rows.append(dict(shape="X32", entry=name, jobs=32, n_in=16, P=P, us_per_launch=us))
        print(f"X32 32 jobs x 16 slots, P {P}: rcmarl_{name:20s} {us:9.1f} us per launch", flush=True)
    return rows


def round_times():
    trs = {name: c2((name, 2.0 if name == "arc_std" else 1.0)) for name in ("arc_std", "gauss")}
    for tr in trs.values():
        tr.rollout_block()
        tr.update_round()
    torch.cuda.synchronize()
    ms = {name: [] for name in trs}
    for _ in range(rounds):
        for name, tr in trs.items():
            tr.rollout_block()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.update_round()
            torch.cuda.synchronize()
            ms[name].append((time.perf_counter() - t0) * 1e3)
    out = {name: dict(median_ms=float(np.median(v)), all_ms=v) for name, v in ms.items()}
    out["added_ms"] = out["arc_std"]["median_ms"] - out["gauss"]["median_ms"]
    print(f"C2 round (arc+clip receivers, {rounds} alternated): arc_std {out['arc_std']['median_ms']:.2f} ms, gauss "
          f"{out['gauss']['median_ms']:.2f} ms ({out['added_ms']:+.3f} ms)", flush=True)
    return out


def main():
    c = card()
    print(c, flush=True)
    result = dict(card=c, c2=c2_launches(), x32=x32(), round=round_times())
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "prof_arc_attack.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
