"""Compare the outputs of the distance-based rules (rcmarl_vector_aggregate), the min-max / min-sum attacks
(rcmarl_adaptive_attack), DnC (rcmarl_dnc_aggregate), nearest-neighbour mixing (rcmarl_nnm_mix), bucketing
(rcmarl_bucket_mix), the tailored attacks (rcmarl_tailored_attack), the subset-selection rules MDA / SMEA
(rcmarl_subset_aggregate), per-neighbour momentum (rcmarl_momentum_mix), the iterative outlier scissor
(rcmarl_ios_aggregate), the pipeline attacks (rcmarl_pipeline_attack), the history attacks (rcmarl_history_attack)
and the IOS-aware attacks (rcmarl_ios_pipeline_attack, rcmarl_ios_history_attack) between two builds of librcmarl.so,
bit for bit.  Their kernels share their bodies with tailored_attack_kernel, pipeline_attack_kernel and history_attack_kernel
(vector_rule, adaptive_gamma, dnc_rule, warp_jacobi, nnm_rows, bucket_draw / bucket_means, tailored_stage /
tailored_range, the candidate search and the momentum step in csrc/train_kernels.cu), so a change there may change
their register allocation and SASS; this shows whether it changed anything they compute.

Each build runs in its own process (RCMARL_LIB selects the library) on the same inputs: 24 messages of 1421 parameters
around a common centre, four of them 1e3 times larger and one holding 1e30; every vector rule at n_in 1 .. 16 (H drawn
per job, repeated in-nodes) with the weights, every min-max / min-sum attack at n_honest 1 .. 16 (scale 1.5, with
gamma), DnC, nnm and bucketing (s = 1, 2, 3) at n_in 1 .. 16 with their weights or mixing matrices, and every tailored
attack x rule at n_in 2 .. 16 (scale 2, with gamma), MDA and SMEA at n_in 1 .. 16 (H drawn per job, with the
weights), momentum at n_in 1 .. 16 over three steps (beta 0.9, the rows and the state after each), IOS at n_in
1 .. 16 (H drawn per job, with the weights), every pipeline
attack x rule (DnC included) x mixing (none, nnm, bucketing at s = 2 with 3 samples) at n_in 2 .. 16 with gamma and
model_out, history_std x rule at n_in 2 .. 16 for (beta, first) = (0.9, 0), (0.99, 0), (0.5, 1), and ios_std in the
pipeline form (mixing none, nnm, bucketing at s = 2) and ios_uv in the history form (beta 0.9) at n_in 2 .. 16 with and
without ARC (H drawn per job), at the trainer's parameter counts.  Entry points a build does not export are skipped when loading it, so a
build from before rcmarl_tailored_attack existed loads too; the outputs of an entry point only one build exports are
listed and not compared.

    python tools/compare_builds.py LIB_A LIB_B [out_dir]     -> prints whether every output is bitwise equal
    (e.g. build the parent commit with `git archive HEAD~1 | tar -x -C DIR && make -C DIR/resilient-consensus-based-marl_b200/csrc`)
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r'''
import ctypes as C, sys
import numpy as np, torch
sys.path[:0] = [sys.argv[2]]
from rcmarl import _lib as L, ops
lib = C.CDLL(L.LIB_PATH)
L.SYMBOLS[:] = [s for s in L.SYMBOLS if hasattr(lib, s[0])]       # an older build lacks the newer entry points
rs = np.random.RandomState(77)
P = 1421
PC = (661, 761, 1101, 1421)
X = (rs.randn(P) + rs.randn(24, P) * rs.uniform(0.05, 1, size=(24, 1))).astype(np.float32)
X[20:] *= 1e3
X[23, 5] = 1e30
msgs = torch.as_tensor(X).cuda()
outs = []
for rule in ("krum", "mkrum", "scclip", "gmed"):
    jobs, dsts, ws = [], [], []
    for n_in in range(1, 17):
        krum = rule in ("krum", "mkrum")
        if krum and n_in < 3:
            continue
        H = int(rs.randint(0, n_in - 2 if krum else n_in))
        d = torch.full((P,), float("nan"), device="cuda")
        w = torch.full((16,), float("nan"), device="cuda")
        nodes = [int(x) for x in rs.choice(24, size=n_in)]
        jobs.append(ops.vector_job(d, msgs, P, PC[n_in % 4], nodes, H, rule, weights_out=w))
        dsts.append(d)
        ws.append(w)
    ops.vector_aggregate(jobs)
    outs += [d.cpu().numpy() for d in dsts] + [w.cpu().numpy() for w in ws]
for a in ("minmax_uv", "minmax_std", "minmax_sgn", "minsum_uv", "minsum_std", "minsum_sgn"):
    jobs, dsts = [], []
    for nh in range(1, 17):
        d = torch.full((P + 1,), float("nan"), device="cuda")
        honest = [int(x) for x in rs.choice(20, size=nh)]
        jobs.append(ops.adaptive_attack_job(d[:P], msgs, P, PC[nh % 4], honest, a, 1.5, gamma_out=d[P:]))
        dsts.append(d)
    ops.adaptive_attack(jobs)
    outs += [d.cpu().numpy() for d in dsts]
if hasattr(lib, "rcmarl_bucket_mix"):
    # nnm and bucketing read their messages and write their rows at one stride: the messages padded to P + 256
    wide = torch.full((24, P + 256), float("nan"), device="cuda")
    wide[:, :P] = msgs
    for kind in ("dnc", "nnm", 1, 2, 3):
        jobs, dsts = [], []
        for n_in in range(1, 17):
            d = torch.full((17, P + 256), float("nan"), device="cuda")
            nodes = [int(x) for x in rs.choice(24, size=n_in)]
            H, n = int(rs.randint(0, n_in)), PC[n_in % 4]
            if kind == "dnc":
                jobs.append(ops.vector_job(d[0], msgs, P, n, nodes, H, L.SPECTRAL_DNC, weights_out=d[16, :16]))
            elif kind == "nnm":
                jobs.append(ops.vector_job(d, wide, P + 256, n, nodes, H, L.MIX_NNM, weights_out=d[16]))
            else:
                jobs.append(ops.bucket_job(d, wide, P + 256, n, nodes, kind, seed=n_in * 977, receiver=n_in, net=n_in & 1,
                                           round=3 * n_in, epoch=n_in % 5, weights_out=d[16]))
            dsts.append(d)
        (ops.dnc_aggregate if kind == "dnc" else ops.nnm_mix if kind == "nnm" else ops.bucket_mix)(jobs)
        outs += [d.cpu().numpy() for d in dsts]
    for rule in ("clip", "trim", "wmsr", "krum", "mkrum", "scclip", "gmed"):
        for a in ("tailored_uv", "tailored_std", "tailored_sgn"):
            jobs, dsts = [], []
            for n_in in range(2, 17):
                if rule in ("krum", "mkrum") and n_in < 3:
                    continue
                n_cr = 1 + n_in % 3 if n_in > 3 else 1
                real = [int(x) for x in rs.choice(24, size=n_in - n_cr)]
                slots = real[:1] + [-1] * n_cr + real[1:]
                honest = [k for k, s in enumerate(slots) if 0 <= s < 20] or [0]
                top = n_in - 3 if rule in ("krum", "mkrum") else (n_in - 1) // 2 if rule == "trim" else n_in - 1
                d = torch.full((P + 1,), float("nan"), device="cuda")
                jobs.append(ops.tailored_attack_job(d[:P], msgs, P, PC[n_in % 4], slots, honest, rule,
                                                    int(rs.randint(0, top + 1)), a, 2.0, gamma_out=d[P:]))
                dsts.append(d)
            ops.tailored_attack(jobs)
            outs += [d.cpu().numpy() for d in dsts]
named = {}
if hasattr(lib, "rcmarl_subset_aggregate"):
    for rule in ("mda", "smea"):
        jobs, dsts = [], []
        for n_in in range(1, 17):
            d = torch.full((P + 16,), float("nan"), device="cuda")
            nodes = [int(x) for x in rs.choice(24, size=n_in)]
            jobs.append(ops.vector_job(d[:P], msgs, P, PC[n_in % 4], nodes, int(rs.randint(0, n_in)),
                                       L.SUBSET_RULES[rule], weights_out=d[P:]))
            dsts.append(d)
        ops.subset_aggregate(jobs)
        named.update({f"subset_{rule}_{k}": d.cpu().numpy() for k, d in enumerate(dsts)})
if hasattr(lib, "rcmarl_momentum_mix"):
    wide = torch.full((24, P + 256), float("nan"), device="cuda")
    wide[:, :P] = msgs
    ref = msgs[0] * 0.5
    Ms = [torch.full((16, P), float("nan"), device="cuda") for _ in range(16)]
    nodes = [[int(x) for x in rs.choice(24, size=n_in)] for n_in in range(1, 17)]
    for step in range(3):
        dsts = [torch.full((16, P + 256), float("nan"), device="cuda") for _ in range(16)]
        ops.momentum_mix([ops.momentum_job(dsts[q], wide, P + 256, PC[(q + 1) % 4], nodes[q], ref, Ms[q], P, 0.9,
                                           int(step == 0)) for q in range(16)])
        named.update({f"momentum_{step}_{q}": np.concatenate([dsts[q].cpu().numpy().ravel(), Ms[q].cpu().numpy().ravel()])
                      for q in range(16)})
if hasattr(lib, "rcmarl_ios_aggregate"):
    jobs, dsts = [], []
    rs_ios = np.random.RandomState(78)                             # its own draws: the later inputs stay the same
    for n_in in range(1, 17):
        d = torch.full((P + 16,), float("nan"), device="cuda")
        nodes = [int(x) for x in rs_ios.choice(24, size=n_in)]
        jobs.append(ops.vector_job(d[:P], msgs, P, PC[n_in % 4], nodes, int(rs_ios.randint(0, n_in)), L.FILTER_IOS,
                                   weights_out=d[P:]))
        dsts.append(d)
    ops.ios_aggregate(jobs)
    named.update({f"ios_{k}": d.cpu().numpy() for k, d in enumerate(dsts)})


def attack_cases(rule):
    """(slots, honest, H, P) of an attack job against `rule` at n_in 2 .. 16, 1-3 crafted slots."""
    out = []
    for n_in in range(2, 17):
        if rule in ("krum", "mkrum") and n_in < 3:
            continue
        n_cr = 1 + n_in % 3 if n_in > 3 else 1
        real = [int(x) for x in rs.choice(20, size=n_in - n_cr, replace=False)]
        slots = real[:1] + [-1] * n_cr + real[1:]
        honest = [k for k, s in enumerate(slots) if 0 <= s < 16] or [0]
        top = n_in - 3 if rule in ("krum", "mkrum") else (n_in - 1) // 2 if rule == "trim" else n_in - 1
        out.append((slots, honest, int(rs.randint(0, top + 1)), PC[n_in % 4]))
    return out


ATTACK_RULES = ("clip", "trim", "wmsr", "krum", "mkrum", "scclip", "gmed", "dnc")
if hasattr(lib, "rcmarl_pipeline_attack"):
    for rule in ATTACK_RULES:
        for mixing in (None, "nnm", ("bucket", 2)):
            for a in ("pipeline_uv", "pipeline_std", "pipeline_sgn"):
                jobs, dsts = [], []
                for slots, honest, H, n in attack_cases(rule):
                    if rule in ("krum", "mkrum") and mixing is not None and len(slots) < 6:
                        continue                                  # too few mixed rows for the rule at H
                    if isinstance(mixing, tuple):
                        n_rows = 1 + (len(slots) - 2) // 2 + 1
                        H = min(H, n_rows - 3 if rule in ("krum", "mkrum") else (n_rows - 1) // 2 if rule == "trim"
                                else n_rows - 1)
                    d = torch.full((2 * P + 1,), float("nan"), device="cuda")
                    jobs.append(ops.pipeline_attack_job(d[:P], msgs, P, n, slots, honest, rule, H, a, 2.0,
                                                        mixing=mixing, n_perms=3, seed=11, attacker=len(slots),
                                                        receiver=2, net=1, round=5, epoch=1, gamma_out=d[2 * P:],
                                                        model_out=d[P:2 * P]))
                    dsts.append(d)
                ops.pipeline_attack(jobs)
                named.update({f"pipeline_{rule}_{mixing}_{a}_{k}": d.cpu().numpy() for k, d in enumerate(dsts)})
if hasattr(lib, "rcmarl_history_attack"):
    ref = msgs[0] * 0.5
    M = (torch.randn(16, P, generator=torch.Generator().manual_seed(5)) * 0.3).cuda()
    for rule in ATTACK_RULES:
        for beta, first in ((0.9, 0), (0.99, 0), (0.5, 1)):
            jobs, dsts = [], []
            for slots, honest, H, n in attack_cases(rule):
                d = torch.full((2 * P + 1,), float("nan"), device="cuda")
                jobs.append(ops.history_attack_job(d[:P], msgs, P, n, slots, honest, rule, H, "history_std", 2.0, ref,
                                                   M, P, beta, first, [slots.index(-1)], gamma_out=d[2 * P:],
                                                   model_out=d[P:2 * P]))
                dsts.append(d)
            ops.history_attack(jobs)
            named.update({f"history_{rule}_{beta}_{first}_{k}": d.cpu().numpy() for k, d in enumerate(dsts)})
if hasattr(lib, "rcmarl_ios_pipeline_attack"):
    rs_att = np.random.RandomState(79)                             # its own draws: the later inputs stay the same
    ref = msgs[0] * 0.5
    M = (torch.randn(16, P, generator=torch.Generator().manual_seed(6)) * 0.3).cuda()
    for arc in (0, 1):
        for mixing in (None, "nnm", ("bucket", 2)):
            jobs, dsts = [], []
            for n_in in range(2, 17):
                n_cr = 1 + n_in % 3 if n_in > 3 else 1
                real = [int(x) for x in rs_att.choice(20, size=n_in - n_cr, replace=False)]
                slots = real[:1] + [-1] * n_cr + real[1:]
                honest = [k for k, s in enumerate(slots) if 0 <= s < 16] or [0]
                n_rows = 1 + (n_in - 2) // 2 + 1 if isinstance(mixing, tuple) else n_in
                n_mixed = n_in if mixing == "nnm" else n_rows - 1 if isinstance(mixing, tuple) else 0
                H, n = int(rs_att.randint(0, n_rows)), PC[n_in % 4]
                if (len(real) + n_mixed + 6 + arc * L.arc_count(H, n_in)) * n > L.PIPELINE_MAX_FLOATS:
                    continue                                      # past the staging bound
                d = torch.full((2 * P + 1,), float("nan"), device="cuda")
                jobs.append(ops.pipeline_attack_job(d[:P], msgs, P, n, slots, honest, "ios", H, "ios_std", 2.0,
                                                    mixing=mixing, n_perms=3, seed=11, attacker=n_in, receiver=2,
                                                    net=1, round=5, epoch=1, gamma_out=d[2 * P:],
                                                    model_out=d[P:2 * P]))
                dsts.append(d)
            ops.ios_pipeline_attack(jobs, arc)
            named.update({f"ios_pipeline_{arc}_{mixing}_{k}": d.cpu().numpy() for k, d in enumerate(dsts)})
        jobs, dsts = [], []
        for n_in in range(2, 17):
            n_cr = 1 + n_in % 3 if n_in > 3 else 1
            real = [int(x) for x in rs_att.choice(20, size=n_in - n_cr, replace=False)]
            slots = real[:1] + [-1] * n_cr + real[1:]
            honest = [k for k, s in enumerate(slots) if 0 <= s < 16] or [0]
            H, n = int(rs_att.randint(0, n_in)), PC[n_in % 4]
            if (n_in + 6 + arc * L.arc_count(H, n_in)) * n > L.HISTORY_MAX_FLOATS:
                continue                                          # past the staging bound
            d = torch.full((2 * P + 1,), float("nan"), device="cuda")
            jobs.append(ops.history_attack_job(d[:P], msgs, P, n, slots, honest, "ios", H, "ios_uv", 2.0, ref, M, P,
                                               0.9, 0, [slots.index(-1)], gamma_out=d[2 * P:], model_out=d[P:2 * P]))
            dsts.append(d)
        ops.ios_history_attack(jobs, arc)
        named.update({f"ios_history_{arc}_{k}": d.cpu().numpy() for k, d in enumerate(dsts)})
np.savez(sys.argv[1], *outs, **named)
'''


def dump(lib, path):
    env = dict(os.environ, RCMARL_LIB=os.path.abspath(lib))
    subprocess.check_call([sys.executable, "-c", CHILD, path, os.path.join(ROOT, "resilient-consensus-based-marl_b200")],
                          env=env)
    return np.load(path)


def main():
    if len(sys.argv) < 3:
        sys.exit(__doc__)
    out_dir = sys.argv[3] if len(sys.argv) > 3 else tempfile.mkdtemp()
    a = dump(sys.argv[1], os.path.join(out_dir, "outputs_a.npz"))
    b = dump(sys.argv[2], os.path.join(out_dir, "outputs_b.npz"))
    common = [k for k in a.files if k in b.files]
    only = sorted(set(a.files) ^ set(b.files))
    diff = [k for k in common if a[k].tobytes() != b[k].tobytes()]
    print(f"{len(common)} output arrays (vector_aggregate, adaptive_attack, dnc_aggregate, nnm_mix, bucket_mix, "
          "tailored_attack, subset_aggregate, momentum_mix, ios_aggregate, pipeline_attack, history_attack, "
          "ios_pipeline_attack and ios_history_attack outputs): "
          + ("bitwise equal" if not diff else f"{len(diff)} differ: {diff[:8]}")
          + (f"; {len(only)} from an entry point only one build exports, not compared" if only else ""))
    sys.exit(1 if diff or not common else 0)


if __name__ == "__main__":
    main()
