"""Launch times of the IOS-aware attacks (rcmarl_ios_pipeline_attack, rcmarl_ios_history_attack), beside the DnC
forms of the base attacks at the same shapes, and the C2 round time on ios_std against gauss, with every cooperative
agent on ios at H = 1:
  C2     6 jobs (3 receivers x 2 nets: P 661 / 761) of 4 slots (3 real, 1 crafted) at H = 1, each of the four forms
         (pipeline, pipeline with ARC, history on momentum 0.9, history with ARC): CUDA events around `reps` launches
         after a warm-up
  X16    30 jobs of 16 slots (15 real, 1 crafted), P 1421, the pipeline form without mixing at H = 3 and H = 7: CUDA
         events around `reps` launches after a warm-up
  round  one C2 update round (two epochs, the benchmark's hyper-parameters) on ios_std (s = 2) and on gauss,
         alternated, `rounds` times each: medians of the host clock around a round that ends in a device synchronise
The card's name and power limit are printed beside the numbers.

    python tools/prof_ios_attack.py [rounds=5] [out_dir]   -> prints one line per measurement (and a JSON file)
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

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


def timed(fn, arr, reps):
    fn(arr)                                    # warm-up: module load and the shared-memory opt-in
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn(arr)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def jobs_for(form, rule, n_jobs, n_in, H, Ps, rs, attack):
    """n_jobs jobs of `form` ("pipeline" / "history") against `rule`, slot n_in - 1 crafted, the rest real."""
    S = max(Ps) + 6
    msgs = torch.as_tensor((rs.randn(1, S) + rs.randn(n_in, S) * 0.5).astype(np.float32)).cuda()
    ref = torch.as_tensor(rs.randn(S).astype(np.float32)).cuda()
    M = torch.as_tensor((rs.randn(n_in, S) * 0.3).astype(np.float32)).cuda()
    dst = torch.zeros(n_jobs, S, device="cuda")
    gam = torch.zeros(n_jobs, 1, device="cuda")
    slots, honest = list(range(n_in - 1)) + [-1], list(range(n_in - 1))
    out = []
    for j in range(n_jobs):
        P = Ps[j % len(Ps)]
        if form == "pipeline":
            out.append(ops.pipeline_attack_job(dst[j], msgs, S, P, slots, honest, rule, H, attack, 2.0,
                                               gamma_out=gam[j]))
        else:
            out.append(ops.history_attack_job(dst[j], msgs, S, P, slots, honest, rule, H, attack, 2.0, ref, M,
                                              S, 0.9, 0, [n_in - 1], gamma_out=gam[j]))
    return ops.job_array(type(out[0]), out), (msgs, ref, M, dst, gam)


# (form, arc) -> (the IOS form, the base entry point of the DnC form at the same staging)
FORMS = {("pipeline", 0): (lambda a: ops.ios_pipeline_attack(a, 0), ops.pipeline_attack),
         ("pipeline", 1): (lambda a: ops.ios_pipeline_attack(a, 1), ops.pipeline_arc_attack),
         ("history", 0): (lambda a: ops.ios_history_attack(a, 0), ops.history_attack),
         ("history", 1): (lambda a: ops.ios_history_attack(a, 1), ops.history_arc_attack)}


def launches(shape, forms, n_jobs, n_in, Hs, Ps, reps, seed):
    rs = np.random.RandomState(seed)
    rows = []
    for H in Hs:
        for form, arc in forms:
            ios, base = FORMS[(form, arc)]
            arr, keep = jobs_for(form, "ios", n_jobs, n_in, H, Ps, rs, "ios_std")
            us = timed(ios, arr, reps)
            darr, dkeep = jobs_for(form, "dnc", n_jobs, n_in, H, Ps, rs, ("arc_" if arc else form + "_") + "std")
            dus = timed(base, darr, reps)
            rows.append(dict(shape=shape, form=form, arc=arc, jobs=n_jobs, n_in=n_in, H=H, P=list(Ps),
                             us_per_launch=us, dnc_us_per_launch=dus))
            print(f"{shape:3s} {form:8s} arc={arc} H {H}: ios {us:10.1f} us, dnc {dus:10.1f} us per launch "
                  f"({n_jobs} jobs, n_in {n_in}, P {'/'.join(map(str, Ps))})", flush=True)
    return rows


def round_times():
    trs = {name: Trainer(**dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"],
                                attack=(name, 2.0 if name == "ios_std" else 1.0), aggregation="ios"))
           for name in ("ios_std", "gauss")}
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
    r = {name: dict(median_ms=float(np.median(v)), all_ms=v) for name, v in ms.items()}
    r["added_ms"] = r["ios_std"]["median_ms"] - r["gauss"]["median_ms"]
    print(f"C2 round (ios receivers, {rounds} alternated): ios_std {r['ios_std']['median_ms']:.2f} ms, "
          f"gauss {r['gauss']['median_ms']:.2f} ms ({r['added_ms']:+.3f} ms)", flush=True)
    return r


def main():
    c = card()
    print(c, flush=True)
    result = dict(card=c, c2=launches("C2", list(FORMS), 6, 4, (1,), (661, 761), 20, 3),
                  x16=launches("X16", [("pipeline", 0)], 30, 16, (3, 7), (1421,), 5, 4), round=round_times())
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "prof_ios_attack.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
