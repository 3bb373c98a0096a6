"""Duration of the one rcmarl_ios_aggregate launch per epoch that Trainer issues for its ios agents, at three team shapes
built from a real Trainer after one update round (its message rows, its receivers' in-nodes with the Byzantine agents'
crafted rows):
  C2      5 agents, agent 4 Byzantine (gauss), 4 cooperative receivers x 2 nets = 8 jobs, n_in 4, P 661 / 761, H 1
  X16 H3  16 agents, 15 cooperative, agent 15 Byzantine, in-neighbourhoods of 16 = 30 jobs, n_in 16, P 1101 / 1421,
          H 3 (3 centre-and-distance passes per job)
  X16 H7  the same at H 7 (7 passes per job)
Reported: the kernel's device time from torch.profiler (mean over launches) and the CUDA-event time per launch of
back-to-back launches (kernel plus launch overhead), with the card's name and power limit.  Each shape is timed over
about one second of launches (at least 3, at most `launches`).

    python tools/prof_ios.py [launches=2000]
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

n_launch = int(sys.argv[1]) if len(sys.argv) > 1 else 2000


def team(name):
    """(Trainer config, H) of the team shape `name` (the shapes of tools/prof_subset.py)."""
    if name == "C2":
        return dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=("gauss", 0.3)), 1
    rs = np.random.RandomState(5)
    NA = 16
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    return dict(labels=["Cooperative"] * 15 + ["Byzantine"], in_nodes=[[(i + k) % NA for k in range(NA)] for i in range(NA)],
                weights=w, desired=rs.randint(0, 10, size=(NA, 2)), nrow=10, ncol=10, n_envs=64, attack=("ipm", 0.5),
                **bench.HYPER), int(name.split("H")[1])


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def timed(arr, count):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(count):
        ops.ios_aggregate(arr)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / count


print(f"{torch.cuda.get_device_name(0)}, power limit {power_limit()}", flush=True)
for name in ("C2", "X16 H3", "X16 H7"):
    cfg, H = team(name.replace(" ", ""))
    n_coop = sum(l == "Cooperative" for l in cfg["labels"])
    tr = Trainer(**dict(cfg, H=H, aggregation=["ios"] * n_coop + ["clip"]))
    tr.rollout_block()
    tr.update_round()
    weights = torch.zeros(2 * n_coop, L.MAX_NEIGHBOURS, device=tr.dev)
    jobs = []
    for q, i in enumerate(tr.ios_agents):              # the job table update_round builds (trainer.py)
        for t, (msgs, P) in enumerate(((tr.msg_c, tr.PC), (tr.msg_t, tr.PT))):
            jobs.append(ops.vector_job(msgs[tr.ios_row[i]], msgs, P, P, tr._receiver_nodes(i), H, L.FILTER_IOS,
                                       weights_out=weights[2 * q + t]))
    arr = ops.job_array(L.VectorJob, jobs)
    ops.ios_aggregate(arr)
    torch.cuda.synchronize()
    first_us = timed(arr, 3)                         # warm, and sizes the timed window to about one second
    count = int(min(n_launch, max(3, 1e6 / max(first_us, 1.0))))
    ev_us = timed(arr, count)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(count):
            ops.ios_aggregate(arr)
        torch.cuda.synchronize()
    k = [e for e in prof.key_averages() if "ios_agg_kernel" in e.key]
    dev_us = (k[0].device_time_total / k[0].count) if k else float("nan")
    n_in = len(tr.in_nodes[tr.ios_agents[0]])
    print(f"{name:6s} ios {len(arr):2d} jobs, n_in {n_in:2d}, H {H}: kernel {dev_us:7.1f} us (profiler), "
          f"{ev_us:7.1f} us per launch back to back (CUDA events, {count} launches)", flush=True)
