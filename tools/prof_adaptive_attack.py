"""Duration of the rcmarl_adaptive_attack launches Trainer issues per epoch for its min-max / min-sum attackers, of
the rcmarl_tailored_attack launches for its tailored attackers and of the rcmarl_pipeline_attack launches for its
pipeline attackers, per attack, at two team shapes built from a real Trainer after one update round (its message rows and its pairs' honest
sets):
  C2   5 agents, agent 4 Byzantine: 3 receivers x 2 nets = 6 jobs, n_honest 3, P 661 / 761
  X16  16 agents, 8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy, circulant in-neighbourhoods of 10: 24 pairs x 2 nets
       = 48 jobs in two launches (32 + 16), n_honest 5, P 1101 / 1421
The tailored attacks are timed at s = 2 against receivers on clip (all three directions) and tailored_std against
receivers on each other rule (the receiver's H is the team's, 1); their cost depends on the rule, gmed costing most.
The pipeline attacks are timed as pipeline_std at s = 2 against receivers on clip and on dnc, each without mixing, with
nnm and with bucketing (s = 2, the trainer's 4 shuffle samples), over min(epochs, 20) epochs (DnC's eigen-solve runs 33
times per job, 132 under bucketing).
Reported per attack: the kernel's device time per epoch from torch.profiler (mean per launch x launches) and the
CUDA-event time per epoch of back-to-back epochs (kernels plus launch overhead), against the same for rcmarl_attack's
gauss on the same job tables.

    python tools/prof_adaptive_attack.py [epochs=200]
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

n_epoch = int(sys.argv[1]) if len(sys.argv) > 1 else 200
ATTACKS = ("minmax_uv", "minmax_std", "minmax_sgn", "minsum_uv", "minsum_std", "minsum_sgn")
# (attack, receiver rule) of the tailored rows
TAILORED = tuple((a, "clip") for a in ("tailored_uv", "tailored_std", "tailored_sgn")) + \
    tuple(("tailored_std", r) for r in ("trim", "wmsr", "krum", "mkrum", "scclip", "gmed"))
# (attack, receiver rule, receiver mixing) of the pipeline rows
PIPELINE = tuple(("pipeline_std", r, m) for r in ("clip", "dnc") for m in (None, "nnm", ("bucket", 2)))
B16 = ["Cooperative", "Byzantine", "Cooperative", "Malicious", "Cooperative", "Byzantine", "Cooperative", "Greedy",
       "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Malicious", "Byzantine", "Cooperative"]


def team(name):
    if name == "C2":
        return dict(bench.workload("C2", 256), labels=["Cooperative"] * 4 + ["Byzantine"], attack=("minmax_std", 1.0))
    rs = np.random.RandomState(5)
    NA = 16
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    return dict(labels=B16, in_nodes=[[(i + k) % NA for k in range(10)] for i in range(NA)], weights=w,
                desired=rs.randint(0, 10, size=(NA, 2)), nrow=10, ncol=10, n_envs=64, H=1, attack=("minmax_std", 1.0),
                **bench.HYPER)


def groups_of(tr, attack, gammas, rule=None, mixing=None):
    """The job tables update_round builds (trainer.py) with every pair on `attack` (a tailored or pipeline one against
    receivers on `rule`, a pipeline one after `mixing`), in groups of MAX_JOBS."""
    jobs = []
    for e, (b, j, honest) in enumerate(tr.byz_pairs):
        for t, (msgs, P) in enumerate(((tr.msg_c, tr.PC), (tr.msg_t, tr.PT))):
            if L.is_pipeline_attack(attack):
                slots, hon = tr._tailored_slots(j)
                jobs.append(ops.pipeline_attack_job(msgs[tr.NA + e], msgs, P, P, slots, hon, rule, tr.H[j], attack, 2.0,
                                                    mixing=mixing, n_perms=L.PIPELINE_PERMS, seed=1, attacker=b,
                                                    receiver=j, net=t, gamma_out=gammas[e, t:t + 1]))
            elif L.is_tailored_attack(attack):
                slots, hon = tr._tailored_slots(j)
                jobs.append(ops.tailored_attack_job(msgs[tr.NA + e], msgs, P, P, slots, hon, rule, tr.H[j], attack, 2.0,
                                                    gamma_out=gammas[e, t:t + 1]))
            elif attack == "gauss":
                jobs.append(ops.attack_job(msgs[tr.NA + e], msgs, P, P, honest, "gauss", 0.3, seed=1, attacker=b, receiver=j))
            else:
                jobs.append(ops.adaptive_attack_job(msgs[tr.NA + e], msgs, P, P, honest, attack, 1.0,
                                                    gamma_out=gammas[e, t:t + 1]))
    cls = L.AttackJob if attack == "gauss" else (L.TailoredAttackJob if L.is_tailored_attack(attack) else
                                                 L.PipelineAttackJob if L.is_pipeline_attack(attack) else L.AdaptiveAttackJob)
    return [ops.job_array(cls, jobs[g:g + L.MAX_JOBS]) for g in range(0, len(jobs), L.MAX_JOBS)]


def epoch(groups, attack):
    launch = ops.attack if attack == "gauss" else (ops.tailored_attack if L.is_tailored_attack(attack) else
                                                    ops.pipeline_attack if L.is_pipeline_attack(attack) else
                                                    ops.adaptive_attack)
    for g in groups:
        launch(g)


def kernel_name(attack):
    if attack == "gauss":
        return "attack_kernel"
    if L.is_pipeline_attack(attack):
        return "pipeline_attack_kernel"
    return "tailored_attack_kernel" if L.is_tailored_attack(attack) else "adaptive_attack_kernel"


print(torch.cuda.get_device_name(0), flush=True)
for name in ("C2", "X16"):
    tr = Trainer(**team(name))
    tr.rollout_block()
    tr.update_round()
    gammas = torch.zeros(len(tr.byz_pairs), 2, device=tr.dev)
    for attack, rule, mixing in tuple((a, None, None) for a in ATTACKS) + (("gauss", None, None),) + \
            tuple(x + (None,) for x in TAILORED) + PIPELINE:
        n_ep = min(n_epoch, 20) if L.is_pipeline_attack(attack) else n_epoch
        groups = groups_of(tr, attack, gammas, rule, mixing)
        for _ in range(2 if L.is_pipeline_attack(attack) else 10):
            epoch(groups, attack)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n_ep):
            epoch(groups, attack)
        b.record()
        torch.cuda.synchronize()
        ev_us = a.elapsed_time(b) * 1e3 / n_ep
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(n_ep):
                epoch(groups, attack)
            torch.cuda.synchronize()
        kname = kernel_name(attack)
        k = [e for e in prof.key_averages() if e.key.split("(")[0].split("::")[-1].split()[-1] == kname]
        dev_us = (k[0].device_time_total / n_ep) if k else float("nan")
        n_jobs = sum(len(g) for g in groups)
        label = attack + (f" vs {rule}" if rule else "") + (f" after {L.mixing_entry(mixing)}" if mixing else "")
        print(f"{name:4s} {label:40s} {n_jobs:2d} jobs in {len(groups)} launch(es), n_honest "
              f"{len(tr.byz_pairs[0][2])}: kernels {dev_us:7.1f} us per epoch (profiler), {ev_us:7.1f} us per epoch back "
              f"to back (CUDA events)", flush=True)
