"""Duration of the one rcmarl_arc_clip launch per epoch that Trainer issues for its cooperative agents that clip
(clipping="arc"), built from a real Trainer after one update round (its message rows and its receivers' in-nodes with
the Byzantine agents' crafted rows):
  C2   5 agents, agent 4 Byzantine (gauss), 4 cooperative receivers x 2 nets = 8 jobs, n_in 4, H 1, P 661 / 761
  X16  16 agents, every one cooperative, in-neighbourhoods of 16 = 32 jobs, n_in 16, H 3, P 1101 / 1421
Reported: the kernel's device time from torch.profiler (mean over launches) and the CUDA-event time per launch of
back-to-back launches (kernel plus launch overhead), with the card's name and power limit.  Then one C2 update round at
the benchmark's 4096 environments, agent 4 Byzantine (gauss), every cooperative agent on clip with and without ARC,
the two trainers alternated round by round (CUDA events around update_round, median of the timed rounds).

    python tools/prof_arc.py [launches=200] [timed_rounds=10]
"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "resilient-consensus-based-marl_b200"))
import bench                                   # noqa: E402
from rcmarl import _lib as L, nets, ops        # noqa: E402
from rcmarl.trainer import Trainer             # noqa: E402

n_launch = int(sys.argv[1]) if len(sys.argv) > 1 else 200
timed_rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 10


def team(name):
    """(Trainer config, H) of the team shape `name`."""
    if name == "C2":
        return dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=("gauss", 0.3)), 1
    rs = np.random.RandomState(5)
    NA = 16
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    return dict(labels=["Cooperative"] * NA, in_nodes=[[(i + k) % NA for k in range(NA)] for i in range(NA)],
                weights=w, desired=rs.randint(0, 10, size=(NA, 2)), nrow=10, ncol=10, n_envs=64, **bench.HYPER), 3


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


print(f"{torch.cuda.get_device_name(0)}, power limit {power_limit()}", flush=True)
for name in ("C2", "X16"):
    cfg, H = team(name)
    tr = Trainer(**dict(cfg, H=H, clipping="arc"))
    tr.rollout_block()
    tr.update_round()
    arr = ops.job_array(L.VectorJob, [                 # the job table update_round builds (trainer.py)
        ops.vector_job(msgs[tr.arc_row[i]], msgs, P, P, tr._momentum_nodes(i), tr.H[i], L.MIX_ARC,
                       weights_out=tr.arc_weights[2 * q + t])
        for q, i in enumerate(tr.arc_agents)
        for t, (msgs, P) in enumerate(((tr.msg_c, tr.PC), (tr.msg_t, tr.PT)))])
    for _ in range(10):
        ops.arc_clip(arr)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n_launch):
        ops.arc_clip(arr)
    b.record()
    torch.cuda.synchronize()
    ev_us = a.elapsed_time(b) * 1e3 / n_launch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n_launch):
            ops.arc_clip(arr)
        torch.cuda.synchronize()
    k = [e for e in prof.key_averages() if "arc_clip_kernel" in e.key]
    dev_us = (k[0].device_time_total / k[0].count) if k else float("nan")
    i0 = tr.arc_agents[0]
    print(f"{name:4s} arc {len(arr):2d} jobs, n_in {len(tr.in_nodes[i0]):2d}, H {H}, P {tr.PC} / {tr.PT}: "
          f"kernel {dev_us:7.1f} us (profiler), {ev_us:7.1f} us per launch back to back (CUDA events)", flush=True)

cfg = dict(bench.workload("C2", 0), labels=["Cooperative"] * 4 + ["Byzantine"], attack=("gauss", 0.3))
trs = {"clip": Trainer(**cfg), "arc+clip": Trainer(**dict(cfg, clipping="arc"))}
ms = {k: [] for k in trs}
for r in range(timed_rounds + 1):
    for k, tr in trs.items():
        tr.rollout_block()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        tr.update_round()
        b.record()
        torch.cuda.synchronize()
        if r > 0:                                       # round 0 warms up
            ms[k].append(a.elapsed_time(b))
med = {k: float(np.median(v)) for k, v in ms.items()}
print(f"C2 update round at {cfg['n_envs']} environments, agent 4 Byzantine (gauss), median of {timed_rounds} alternated: "
      f"clip {med['clip']:.2f} ms, arc+clip {med['arc+clip']:.2f} ms ({med['arc+clip'] - med['clip']:+.3f} ms); "
      f"launches per round {trs['clip'].launches // (timed_rounds + 1)} / "
      f"{trs['arc+clip'].launches // (timed_rounds + 1)}", flush=True)
