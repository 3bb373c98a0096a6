"""Kernel time per launch of rcmarl_history_attack as Trainer issues it, at two team shapes, with every cooperative agent
on momentum at beta = 0.9 before clip, gmed (a distance-based rule) and dnc, every Byzantine agent on history_std at
s = 2:
  C2   5 agents, agent 4 Byzantine: 3 receivers x 2 nets = 6 jobs in one launch, n_in 4, P 661 / 761
  X16  16 agents, 8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy, circulant in-neighbourhoods of 10: 24 pairs x 2
       nets = 48 jobs in two launches (32 + 16), n_in 10, P 1101 / 1421
Each shape runs one warm-up update round, then `rounds` profiled rounds; the kernel's device time per launch is the mean
over the profiled launches of history_attack_kernel (torch.profiler, CUDA activities), beside that of momentum_mix_kernel
in the same rounds.

    python tools/prof_history_attack.py [rounds=2] [out_dir]   -> prints one line per shape x rule (and a JSON file)
"""
import json
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "resilient-consensus-based-marl_b200"))
import bench                                   # noqa: E402
from rcmarl import nets                        # noqa: E402
from rcmarl.trainer import Trainer             # noqa: E402

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 2
out_dir = sys.argv[2] if len(sys.argv) > 2 else None
B16 = ["Cooperative", "Byzantine", "Cooperative", "Malicious", "Cooperative", "Byzantine", "Cooperative", "Greedy",
       "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Malicious", "Byzantine", "Cooperative"]
ATTACK = ("history_std", 2.0)


def team(name):
    if name == "C2":
        return dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=ATTACK)
    rs = np.random.RandomState(5)
    NA = 16
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    return dict(labels=B16, in_nodes=[[(i + k) % NA for k in range(10)] for i in range(NA)], weights=w,
                desired=rs.randint(0, 10, size=(NA, 2)), nrow=10, ncol=10, n_envs=64, H=1, attack=ATTACK,
                **bench.HYPER)


def kernel_us(prof, name):
    """(mean device time per launch in us, launches) of the kernels whose name contains `name`."""
    ev = [e for e in prof.events() if name in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    if not ev:
        return None, 0
    return float(np.mean([e.device_time_total for e in ev])), len(ev)


def main():
    dev = torch.cuda.get_device_name(0)
    result = dict(card=dev, beta=0.9, attack=list(ATTACK), rows=[])
    for shape in ("C2", "X16"):
        for rule in ("clip", "gmed", "dnc"):
            tr = Trainer(**dict(team(shape), aggregation=rule, momentum=0.9))
            tr.rollout_block()
            tr.update_round()                                       # warm-up: first steps, module loads
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(rounds):
                    tr.rollout_block()
                    tr.update_round()
                torch.cuda.synchronize()
            us, n = kernel_us(prof, "history_attack_kernel")
            mom, _ = kernel_us(prof, "momentum_mix_kernel")
            jobs = 2 * len(tr.hist_pairs)
            row = dict(shape=shape, rule=rule, jobs=jobs, launches=n, us_per_launch=us, momentum_us_per_launch=mom)
            result["rows"].append(row)
            print(f"{dev} {shape:3s} m0.9+{rule:5s} {jobs:2d} jobs: history_attack_kernel {us:9.1f} us per launch "
                  f"({n} launches), momentum_mix_kernel {mom:6.1f} us", flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "prof_history_attack.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
