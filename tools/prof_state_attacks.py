"""Duration of one rcmarl_dissensus_attack and one rcmarl_mimic_attack launch, at two team shapes built from a real
Trainer after one update round (its message rows and its pairs' honest sets):
  C2   5 agents, agent 4 Byzantine: 3 receivers x 2 nets = 6 jobs, n_honest 3, P 661 / 761
  X16  16 agents, 8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy, circulant in-neighbourhoods of 10: the first 16
       pairs x 2 nets = 32 jobs in one launch, n_honest 5, P 1101 / 1421
The mimic launch is timed with a power step (update = 1, the first T0 epochs) and without one (update = 0, the frozen
direction).  Reported per launch: the kernel's device time from torch.profiler (mean over launches) and the CUDA-event
time of back-to-back launches (kernel plus launch overhead), against the same for rcmarl_attack's gauss on the same
pairs.

    python tools/prof_state_attacks.py [launches=500]
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "resilient-consensus-based-marl_b200"))
import bench                                   # noqa: E402
from rcmarl import _lib as L, nets, ops        # noqa: E402
from rcmarl.trainer import Trainer             # noqa: E402

n_launch = int(sys.argv[1]) if len(sys.argv) > 1 else 500
B16 = ["Cooperative", "Byzantine", "Cooperative", "Malicious", "Cooperative", "Byzantine", "Cooperative", "Greedy",
       "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Malicious", "Byzantine", "Cooperative"]


def team(name):
    if name == "C2":
        return dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=("mimic", 50))
    rs = np.random.RandomState(5)
    NA = 16
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    return dict(labels=B16, in_nodes=[[(i + k) % NA for k in range(10)] for i in range(NA)], weights=w,
                desired=rs.randint(0, 10, size=(NA, 2)), nrow=10, ncol=10, n_envs=64, H=1, attack=("mimic", 50),
                **bench.HYPER)


def jobs_of(tr, attack, z, tgt, update):
    """One job array of at most MAX_JOBS jobs (the first pairs, both nets) for `attack`, as update_round builds them."""
    jobs = []
    for e, (b, j, honest) in enumerate(tr.byz_pairs[:L.MAX_JOBS // 2]):
        for t, (msgs, P) in enumerate(((tr.msg_c, tr.PC), (tr.msg_t, tr.PT))):
            if attack == "dissensus":
                jobs.append(ops.dissensus_attack_job(msgs[tr.NA + e], msgs, P, P, j, honest, 1, 1.0))
            elif attack == "mimic":
                cand = [k for k, i in enumerate(honest) if i != j] or list(range(len(honest)))
                jobs.append(ops.mimic_attack_job(msgs[tr.NA + e], msgs, P, P, honest, cand, z[e, t], update,
                                                 target_out=tgt[e, t:t + 1]))
            else:
                jobs.append(ops.attack_job(msgs[tr.NA + e], msgs, P, P, honest, "gauss", 0.3, seed=1, attacker=b, receiver=j))
    cls = {"dissensus": L.DissensusJob, "mimic": L.MimicJob}.get(attack, L.AttackJob)
    return ops.job_array(cls, jobs)


LAUNCH = {"dissensus": ops.dissensus_attack, "mimic": ops.mimic_attack, "gauss": ops.attack}
KERNEL = {"dissensus": "dissensus_attack_kernel", "mimic": "mimic_attack_kernel", "gauss": "attack_kernel"}

print(torch.cuda.get_device_name(0), flush=True)
for name in ("C2", "X16"):
    tr = Trainer(**team(name))
    tr.rollout_block()
    tr.update_round()
    z = torch.zeros(len(tr.byz_pairs), 2, tr.PT, device=tr.dev)
    tgt = torch.zeros(len(tr.byz_pairs), 2, dtype=torch.int32, device=tr.dev)
    for attack, update in (("gauss", 0), ("dissensus", 0), ("mimic", 1), ("mimic", 0)):
        arr = jobs_of(tr, attack, z, tgt, update)
        launch = LAUNCH[attack]
        for _ in range(20):
            launch(arr)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n_launch):
            launch(arr)
        b.record()
        torch.cuda.synchronize()
        ev_us = a.elapsed_time(b) * 1e3 / n_launch
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(n_launch):
                launch(arr)
            torch.cuda.synchronize()
        k = [e for e in prof.key_averages() if e.key.split("(")[0].split("::")[-1].split()[-1] == KERNEL[attack]]
        dev_us = (k[0].device_time_total / n_launch) if k else float("nan")
        label = attack + (f" (update {update})" if attack == "mimic" else "")
        print(f"{name:4s} {label:18s} {len(arr):2d} jobs, n_honest {len(tr.byz_pairs[0][2])}: kernel {dev_us:7.1f} us "
              f"per launch (profiler), {ev_us:7.1f} us per launch back to back (CUDA events)", flush=True)
