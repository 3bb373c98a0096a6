"""CPU checks of the IOS-aware Byzantine messages (rcmarl_ios_pipeline_attack, rcmarl_ios_history_attack,
include/rcmarl.h): the oracle (tests/ios_attack_oracle.py) at H = 0, where IOS is the plain mean and the craft is the
DnC craft at H = 0, and at H = n_rows - 1, where IOS keeps one row; the constants, prototypes and struct sizes as gcc
sees the header; the library's refusals, read in a child process that sees no device (a table that passes every check
reaches the CUDA runtime and comes back RCMARL_ERR_CUDA, a refused one RCMARL_ERR_ARG); the attack names and bindings;
and the Trainer's routing, refusals and every field of the jobs it builds for its IOS pairs."""
import ctypes
import functools
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import history_attack_oracle as HO
import ios_attack_oracle as IAO
import ios_oracle as IO
import pipeline_attack_oracle as PA
import subset_attack_oracle as SAO
import test_arc_attack_cpu as AC
import test_history_attack_cpu as HC
import test_subset_attack_cpu as SC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
SLOTS, HONEST = HC.SLOTS, HC.HONEST
no_device, built, C5, BYZ = HC.no_device, HC.built, HC.C5, HC.BYZ
ERR_ARG, ERR_CUDA = -1, -3


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("mixing", [None, "nnm", ("bucket", 2)])
@pytest.mark.parametrize("arc", [False, True])
def test_at_h0_the_pipeline_form_is_the_dnc_pipeline_oracle(mixing, arc):
    rs = np.random.RandomState(17100 + 2 * arc)
    X = HC._stack(rs, dtype=np.float64)
    for d in ("uv", "std", "sgn"):
        m, g, O, R, _ = IAO.craft_pipeline(X, SLOTS, HONEST, "ios", 0, "ios_" + d, 2.0, mixing=mixing, n_perms=2,
                                           arc=arc)
        if arc:     # at H = 0 ARC is the identity: the pipeline craft
            pm, pg, pO, pR, _ = SAO.craft_pipeline(X, SLOTS, HONEST, "dnc", 0, "subset_" + d, 2.0, mixing=mixing,
                                                   n_perms=2, arc=True)
        else:
            pm, pg, pO, pR = PA.craft(X, SLOTS, HONEST, "dnc", 0, "pipeline_" + d, 2.0, mixing=mixing, n_perms=2)
        assert np.array_equal(m, pm) and g == pg and np.array_equal(O, pO) and np.array_equal(R, pR)


@pytest.mark.parametrize("dtype", [np.float64, f32])
def test_at_h0_the_history_form_is_the_dnc_history_oracle(dtype):
    rs = np.random.RandomState(17200)
    X = HC._stack(rs, dtype=dtype)
    c = (X[0] + rs.randn(X.shape[1]) * 0.1).astype(dtype)
    M = (rs.randn(len(SLOTS), X.shape[1]) * 0.2).astype(dtype)
    for d in ("uv", "std", "sgn"):
        m, g, O, R, _ = IAO.craft_history(X, SLOTS, HONEST, "ios", 0, "ios_" + d, 2.0, c, M, 0.9, False, [1, 4])
        hm, hg, hO, hR, _ = HO.craft(X, SLOTS, HONEST, "dnc", 0, "history_" + d, 2.0, c, M, 0.9, False, [1, 4])
        assert np.array_equal(m, hm) and g == hg and np.array_equal(O, hO) and np.array_equal(R, hR)


@pytest.mark.parametrize("arc", [False, True])
def test_at_the_largest_h_the_rule_keeps_one_row(arc):
    """H = n_rows - 1: IOS keeps exactly one row, so R is bitwise one of the rule's rows at every candidate."""
    rs = np.random.RandomState(17300 + arc)
    X = HC._stack(rs, dtype=np.float64)
    n = len(SLOTS)
    m, g, O, R, _ = IAO.craft_pipeline(X, SLOTS, HONEST, "ios", n - 1, "ios_std", 2.0, arc=arc)
    Y = SAO._clip(np.stack([m if s < 0 else X[s] for s in SLOTS]), n - 1, arc)
    (k,) = IO.kept(Y, n - 1)
    assert np.array_equal(R, Y[k])
    c = (X[0] + rs.randn(X.shape[1]) * 0.1).astype(np.float64)
    m, g, O, R, _ = IAO.craft_history(X, SLOTS, HONEST, "ios", n - 1, "ios_uv", 2.0, c, None, 0.9, True, [1, 4],
                                      arc=arc)
    rows = [HO.step_row(X[s], c, None, 0.9, True) for s in SLOTS if s >= 0] + [HO.step_row(m, c, None, 0.9, True)]
    assert any(np.array_equal(R, r) for r in rows)
    m, g, O, R, _ = IAO.craft_pipeline(X, SLOTS, HONEST, "ios", 3, "ios_std", 2.0, mixing=("bucket", 3), n_perms=2,
                                       arc=arc)                                  # 1 + ceil(7 / 3) = 4 rows, H = 4 - 1
    assert R.shape == X[0].shape
    with pytest.raises(ValueError):
        IAO.craft_pipeline(X, [-1] + SLOTS[1:], HONEST[1:], "ios", 1, "ios_std", 2.0, arc=True)   # crafted slot 0


def test_against_other_rules_the_oracle_is_the_subset_oracle():
    rs = np.random.RandomState(17400)
    X = HC._stack(rs, dtype=np.float64)
    for rule in ("mda", "smea", "clip", "dnc", "krum"):
        got = IAO.craft_pipeline(X, SLOTS, HONEST, rule, 1, "ios_sgn", 1.5, mixing="nnm")
        want = SAO.craft_pipeline(X, SLOTS, HONEST, rule, 1, "subset_sgn", 1.5, mixing="nnm")
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), rule


# ------------------------------------------------------------------------------------------------ C ABI
def test_constants_prototypes_and_struct_sizes_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "ios.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*p)(const rcmarl_pipeline_attack_job*, int, int, void*) = rcmarl_ios_pipeline_attack;'
                   'int (*h)(const rcmarl_history_attack_job*, int, int, void*) = rcmarl_ios_history_attack;'
                   'printf("%d %d %d %d %zu %zu %zu\\n", (int)RCMARL_TAILOR_FILTER, (int)RCMARL_TAILOR_SUBSET, '
                   '(int)RCMARL_FILTER_IOS, (int)RCMARL_PIPELINE_MAX_FLOATS, sizeof(rcmarl_tailored_attack_job), '
                   'sizeof(rcmarl_pipeline_attack_job), sizeof(rcmarl_history_attack_job));'
                   'return (p(0, 0, 0, 0) | h(0, 0, 0, 0)) ? 1 : 0;}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\n'
                    'int rcmarl_ios_pipeline_attack(const rcmarl_pipeline_attack_job* j, int n, int a, void* s)'
                    '{(void)j; (void)n; (void)a; (void)s; return 0;}\n'
                    'int rcmarl_ios_history_attack(const rcmarl_history_attack_job* j, int n, int a, void* s)'
                    '{(void)j; (void)n; (void)a; (void)s; return 0;}')
    exe = tmp_path / "ios"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    fam, sub, rule, bound, st, sp, sh = map(int, subprocess.check_output([str(exe)], text=True).split())
    assert (fam, sub, rule, bound) == (L.TAILOR_FILTER, L.TAILOR_SUBSET, L.FILTER_IOS, L.PIPELINE_MAX_FLOATS) \
        == (4, 3, 0, 37 * 1421)
    assert (st, sp, sh) == (ctypes.sizeof(L.TailoredAttackJob), ctypes.sizeof(L.PipelineAttackJob),
                            ctypes.sizeof(L.HistoryAttackJob))
    # the 227 KB a CTA may opt in to holds the bounds and the IOS instantiations' static shared memory (ptxas -v: at
    # most 3 040 B in the pipeline form, 1 824 B in the history form)
    assert L.PIPELINE_MAX_FLOATS * 4 + 3040 <= 227 * 1024 and L.HISTORY_MAX_FLOATS * 4 + 1824 <= 227 * 1024
    lib = L.lib()
    assert lib.rcmarl_ios_pipeline_attack.argtypes == [ctypes.POINTER(L.PipelineAttackJob), ctypes.c_int,
                                                       ctypes.c_int, L.c_fp]
    assert lib.rcmarl_ios_history_attack.argtypes == [ctypes.POINTER(L.HistoryAttackJob), ctypes.c_int,
                                                      ctypes.c_int, L.c_fp]
    assert lib.rcmarl_ios_pipeline_attack.restype == lib.rcmarl_ios_history_attack.restype == ctypes.c_int


# A case is (entry, arc, form, job fields): form "pipeline" builds test_arc_attack_cpu._pjob, "history"
# test_history_attack_cpu._job, each with family FILTER and rule IOS unless the fields say otherwise.  Two tables are
# passed per case: the job alone and the job behind a valid one.
def _jobs(form, fields):
    from rcmarl import _lib as L
    kw = dict(family=L.TAILOR_FILTER, rule=L.FILTER_IOS)
    kw.update(fields)
    if form == "pipeline":
        mixing = kw.pop("mixing", 0)
        s = kw.pop("s", 2)
        j = AC._pjob(mixing=mixing, **kw)
        j.s = s
        other = AC._pjob(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000,
                         family=L.TAILOR_FILTER, rule=L.FILTER_IOS)
        return L.PipelineAttackJob, [j], [other, j]
    other = HC._job(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000,
                    family=L.TAILOR_FILTER, rule=L.FILTER_IOS)
    j = HC._job(**kw)
    return L.HistoryAttackJob, [j], [other, j]


def _codes(cases):
    """The return codes of every case's two tables, in a child process that sees no device."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = ("import json, sys; sys.path[:0] = sys.argv[2:]; import test_ios_attack_cpu as T; "
            "print(json.dumps(T._run([tuple(c) for c in json.loads(sys.argv[1])])))")
    paths = [os.path.dirname(os.path.abspath(__file__)), ROOT, os.path.join(ROOT, "resilient-consensus-based-marl_b200")]
    out = subprocess.run([sys.executable, "-c", code, json.dumps(cases)] + paths, env=env, capture_output=True,
                         text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def _run(cases):
    from rcmarl import _lib as L
    lib = L.lib()
    codes = []
    for entry, arc, form, fields in cases:
        cls, *tables = _jobs(form, fields)
        codes.append([getattr(lib, entry)((cls * len(t))(*t), len(t), arc, None) for t in tables])
    return codes


# the base refusals other than the family (HC.BAD[10]); the pipeline form's staging at HC.BAD[33]'s n fits its bound
PIPE_BAD = [b for b in HC.BAD[:22] + HC.BAD[34:37] if b != dict(family=3)]
HIST_BAD = [b for b in HC.BAD if b != dict(family=3)]
IOS_BAD = [dict(family=0), dict(family=1), dict(family=2), dict(family=3), dict(family=5), dict(rule=1),
           dict(rule=-1), dict(H=-1), dict(H=4)]


def test_refusals_without_a_device():
    from rcmarl import _lib as L
    R, NN = "rcmarl_ios_pipeline_attack", "rcmarl_ios_history_attack"
    big = dict(n_in=16, slots=list(range(15)) + [-1], honest_mask=(1 << 15) - 1, msg_stride=2000, dst=1 << 28,
               gamma_out=1 << 27, model_out=(1 << 27) + 64)
    hist_big = dict(big, momentum_stride=2000, own_mask=1 << 15)
    far = dict(dst=1 << 28, gamma_out=1 << 27, model_out=(1 << 27) + 64)
    admitted = [
        (R, 0, "pipeline", {}), (R, 1, "pipeline", {}), (NN, 0, "history", {}), (NN, 1, "history", {}),
        (R, 0, "pipeline", dict(mixing=L.PIPE_NNM)),
        (R, 1, "pipeline", dict(mixing=L.PIPE_BUCKET, H=2)),            # rows: own + 2 bucket means, H < 3
        (R, 0, "pipeline", dict(H=3)), (NN, 1, "history", dict(H=3)),
        (NN, 0, "history", dict(far, n=22 * 1421 // 10)),               # (4 + 6) * n at the bound
        # at the bounds: 16 slots, 15 real, n = 1421 (the 16-agent team-reward net)
        (R, 0, "pipeline", dict(big, n=1421, H=7, mixing=L.PIPE_NNM)),  # 15 + 16 + 6 = 37 rows
        (R, 1, "pipeline", dict(big, n=1421, H=8, mixing=L.PIPE_BUCKET)),   # 15 + 8 + 6 + k_clip 8 = 37 rows
        (R, 1, "pipeline", dict(big, n=1421, H=1, mixing=L.PIPE_BUCKET, s=1)),   # 15 + 15 + 6 + k_clip 1 = 37 rows
        (R, 1, "pipeline", dict(big, n=1421, H=15)),                    # 15 + 6 + k_clip 1
        (NN, 0, "history", dict(hist_big, n=1421, H=7)),                # 16 + 6 = 22 rows
        (NN, 1, "history", dict(hist_big, n=1421, H=0)),                # k_clip 0
    ]
    refused = [(R, 0, "pipeline", b) for b in PIPE_BAD + IOS_BAD] + [
        (NN, 0, "history", b) for b in HIST_BAD + IOS_BAD] + [
        (R, 2, "pipeline", {}), (R, -1, "pipeline", {}), (NN, 2, "history", {}),
        (R, 1, "pipeline", dict(slots=[-1, 1, 2, 3], honest_mask=0b1010)),       # arc = 1, a crafted slot 0
        (NN, 1, "history", dict(slots=[-1, 1, 2, 3], honest_mask=0b1010, own_mask=0b0001)),
        (R, 0, "pipeline", dict(mixing=L.PIPE_BUCKET, H=3)),            # H outside [0, n_rows = 3)
        (R, 0, "pipeline", dict(mixing=3)), (R, 0, "pipeline", dict(mixing=L.PIPE_BUCKET, s=0)),
        (NN, 0, "history", dict(far, n=22 * 1421 // 10 + 1)),
        # one row of floats past the bounds
        (R, 0, "pipeline", dict(big, n=1422, H=7, mixing=L.PIPE_NNM)),
        (R, 1, "pipeline", dict(big, n=1421, H=1, mixing=L.PIPE_NNM)),  # 37 rows + k_clip 1
        (R, 1, "pipeline", dict(big, n=1422, H=8, mixing=L.PIPE_BUCKET)),
        (R, 1, "pipeline", dict(big, n=1421, H=2, mixing=L.PIPE_BUCKET, s=1)),   # 36 rows + k_clip 3
        (NN, 0, "history", dict(hist_big, n=1422, H=7)),
        (NN, 1, "history", dict(hist_big, n=1421, H=1)),                # 22 rows + k_clip 1
    ]
    codes = _codes(admitted + refused)
    for case, got in zip(admitted, codes[:len(admitted)]):
        assert got == [ERR_CUDA, ERR_CUDA], case
    for case, got in zip(refused, codes[len(admitted):]):
        assert got == [ERR_ARG, ERR_ARG], case


def test_the_other_entry_points_refuse_family_filter_and_bad_job_counts():
    from rcmarl import _lib as L
    lib = L.lib()
    p = AC._pjob(family=L.TAILOR_FILTER, rule=L.FILTER_IOS)
    h = HC._job(family=L.TAILOR_FILTER, rule=L.FILTER_IOS)
    for fn in (lib.rcmarl_pipeline_attack, lib.rcmarl_pipeline_arc_attack):
        assert fn((L.PipelineAttackJob * 1)(p), 1, None) == ERR_ARG
    for fn in (lib.rcmarl_history_attack, lib.rcmarl_history_arc_attack):
        assert fn((L.HistoryAttackJob * 1)(h), 1, None) == ERR_ARG
    t = L.TailoredAttackJob.from_buffer_copy(h.attack)
    assert lib.rcmarl_tailored_attack((L.TailoredAttackJob * 1)(t), 1, None) == ERR_ARG
    for arc in (0, 1):
        assert lib.rcmarl_subset_pipeline_attack((L.PipelineAttackJob * 1)(p), 1, arc, None) == ERR_ARG
        assert lib.rcmarl_subset_history_attack((L.HistoryAttackJob * 1)(h), 1, arc, None) == ERR_ARG
        assert lib.rcmarl_ios_pipeline_attack(None, 1, arc, None) == ERR_ARG
        assert lib.rcmarl_ios_history_attack(None, 1, arc, None) == ERR_ARG
        arr = (L.HistoryAttackJob * 33)(*[HC._job(dst=(1 << 26) + 4 * 1000 * i, gamma_out=(1 << 27) + 4 * i,
                                                  model_out=(1 << 28) + 4 * 1000 * i, family=L.TAILOR_FILTER,
                                                  rule=L.FILTER_IOS) for i in range(33)])
        assert lib.rcmarl_ios_history_attack(arr, 0, arc, None) == ERR_ARG
        assert lib.rcmarl_ios_history_attack(arr, 33, arc, None) == ERR_ARG


def test_attack_names_and_bindings():
    import torch
    from rcmarl import _lib as L, ops
    assert sorted(L.IOS_ATTACKS) == ["ios_sgn", "ios_std", "ios_uv"]
    for d, dev in (("uv", 0), ("std", 1), ("sgn", 2)):
        kind, param = L.check_attack((f"ios_{d}", 2))
        assert isinstance(kind, L.IosAttackKind) and int(kind) == dev and param == 2.0
        assert not isinstance(kind, (L.SubsetAttackKind, L.ArcAttackKind, L.HistoryKind, L.PipelineKind,
                                     L.TailoredKind))
        assert L.is_ios_attack(f"ios_{d}") and not L.is_subset_attack(f"ios_{d}") and not L.is_ios_attack(d)
    assert L.check_attack(("ios_std", 0.0))[1] == 0.0
    for bad in (("ios_uv", -0.5), ("ios_std", float("nan")), ("ios_sgn", float("inf")), ("ios", 1.0),
                ("ios_ios", 1.0)):
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)
    x = torch.zeros(8, 50)
    M = torch.zeros(4, 60)
    j = ops.history_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "ios", 1, "ios_sgn", 1.5, x[6], M, 60, 0.9, 1,
                               [2])
    assert (j.attack.family, j.attack.rule, j.attack.dev, j.attack.scale) == (L.TAILOR_FILTER, L.FILTER_IOS,
                                                                              L.DEV_SGN, 1.5)
    j = ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "ios", 1, "ios_uv", 1.0, mixing="nnm")
    assert (j.attack.family, j.attack.rule, j.attack.dev, j.mixing) == (L.TAILOR_FILTER, L.FILTER_IOS, L.DEV_UV,
                                                                        L.PIPE_NNM)
    # against mda / smea an IOS name builds the subset attack's job, against any other rule the ARC attack's
    for rule in ("mda", "smea", "dnc", "krum", "clip"):
        a = ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], rule, 1, "ios_uv", 1.0)
        b = ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], rule, 1, "subset_uv", 1.0)
        assert (a.attack.family, a.attack.rule, a.attack.dev) == (b.attack.family, b.attack.rule, b.attack.dev), rule
    for name in ("subset_uv", "arc_uv", "pipeline_uv"):     # other names never map ios
        with pytest.raises(Exception):
            ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "ios", 1, name, 1.0)
    with pytest.raises(L.RcmarlError, match="ios_uv"):
        ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "ios", 1, "ios_bogus", 1.0)
    assert callable(ops.ios_pipeline_attack) and callable(ops.ios_history_attack)


# ------------------------------------------------------------------------------------------------ Trainer
def trainer(aggregation, momentum=None, clipping=None, attack=("ios_std", 2.0), mixing=None, H=1, **kw):
    from rcmarl.trainer import Trainer
    return Trainer(labels=BYZ, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing, momentum=momentum, clipping=clipping, **kw)


@pytest.mark.parametrize("aggregation,momentum,mixing,clipping", [
    ("ios", None, None, None), ("ios", 0.9, None, "arc"), ("ios", None, "nnm", "arc"), ("ios", None, ("bucket", 2), None),
    ("mda", 0.9, None, "arc"), ("clip", None, None, "arc"), ("dnc", 0.9, None, None),
    (["ios", "smea", "krum", "ios", "clip"], [None, 0.9, None, 0.9, None], [None, None, "nnm", None, None],
     ["arc", None, None, "arc", None]),
])
def test_trainer_accepts_ios_attackers(no_device, aggregation, momentum, mixing, clipping):
    for attack in (("ios_std", 2.0), ("ios_uv", 1.0), ("ios_sgn", 0.0)):
        with pytest.raises(no_device) as ex:
            trainer(aggregation, momentum, clipping, attack=attack, mixing=mixing)
        tr = built(ex)
        assert tr.ios_pairs == [0, 1, 2] and tr.gamma_pairs == [0, 1, 2]
        assert tr.subset_pairs == tr.arc_pairs == tr.hist_pairs == []


def test_trainer_accepts_ios_attackers_beside_older_attackers(no_device):
    """A mixed team: one ios_* attacker and one subset_* attacker, against ios, mda and clip receivers; the subset
    attacker only hears receivers that are not on ios."""
    from rcmarl.trainer import Trainer
    labels = ["Cooperative"] * 4 + ["Byzantine"] * 2
    in_nodes = [[0, 1, 4, 3], [1, 2, 4, 5], [2, 3, 5, 0], [3, 0, 4, 1], [4, 0, 1, 2], [5, 0, 1, 2]]
    with pytest.raises(no_device) as ex:
        Trainer(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((6, 2)), H=1,
                aggregation=["ios", "mda", "clip", "ios", "clip", "clip"], clipping=["arc"] + [None] * 5,
                attack=[None] * 4 + [("ios_std", 2.0), ("subset_uv", 1.0)])
    tr = built(ex)
    assert [tr.byz_pairs[e][:2] for e in tr.ios_pairs] == [(4, 0), (4, 1), (4, 3)]
    assert [tr.byz_pairs[e][:2] for e in tr.subset_pairs] == [(5, 1), (5, 2)]
    assert tr.gamma_pairs == tr.subset_pairs + tr.ios_pairs


@pytest.mark.parametrize("name", ["tailored_std", "pipeline_uv", "history_sgn", "arc_std", "subset_uv"])
def test_older_adaptive_attacks_stay_refused_against_ios(no_device, name):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="attack against agent .*'ios' the attack does not model"):
        trainer("ios", clipping="arc" if name in ("arc_std", "subset_uv") else None, attack=(name, 2.0))


def test_trainer_refuses_a_job_past_the_staging_bound(no_device):
    """16 agents in one clique of 16 on ios, nnm and ARC at H = 1 (k_clip = 1): (15 + 16 + 6 + 1) * 1421 > 37 * 1421;
    without ARC (37 rows) the job fits."""
    from rcmarl import _lib as L
    from rcmarl.trainer import Trainer
    labels = ["Cooperative"] * 15 + ["Byzantine"]
    in_nodes = [[i] + [k for k in range(16) if k != i] for i in range(16)]
    kw = dict(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((16, 2)), aggregation="ios",
              mixing="nnm", attack=[None] * 15 + [("ios_std", 2.0)], H=1)
    with pytest.raises(L.RcmarlError, match="an IOS attack against agent 0, whose job stages 53998 floats, more than "
                                            "the 52577 the library admits"):
        Trainer(clipping="arc", **kw)
    with pytest.raises(no_device):
        Trainer(**kw)
    with pytest.raises(L.RcmarlError, match="an IOS attack against agent 0, whose job stages 32683 floats, more than "
                                            "the 31262 the library admits"):
        Trainer(**dict(kw, mixing=None, momentum=0.9, clipping="arc"))   # (16 + 6 + 1) * 1421 > 22 * 1421


def test_job_layout_against_ios_and_other_receivers(monkeypatch):
    """Attackers 4 (ios_std) and 5 (ios_uv; receiver 2 lists 4 twice) against receivers 0 (ios, clips), 1 (ios, nnm),
    2 (ios, momentum, clips), 3 (ios, bucketing), 6 (mda, momentum) and 7 (clip, clips): every field of every job, the
    launch each group goes to and the momentum index of each history-form job; the jobs against the receivers on mda
    and clip are field for field a subset_* pair's."""
    from rcmarl import _lib as L, ops
    labels = ["Cooperative"] * 4 + ["Byzantine"] * 2 + ["Cooperative"] * 2
    in_nodes = [[0, 1, 4, 3], [1, 2, 4, 5], [2, 4, 3, 4, 5], [3, 0, 5, 1], [4, 0, 1, 2], [5, 0, 1, 2], [6, 5, 0, 1],
                [7, 4, 0, 1]]
    agg = ["ios", "ios", "ios", "ios", "clip", "clip", "mda", "clip"]
    mom = [None, None, 0.9, None, None, None, 0.5, None]
    mixing = [None, "nnm", None, ("bucket", 2), None, None, None, None]
    clip = ["arc", None, "arc", None, None, None, None, "arc"]
    kw = dict(labels=labels, in_nodes=in_nodes, desired=np.zeros((8, 2)), momentum=mom, mixing=mixing, clipping=clip,
              aggregation=agg)
    tr = AC._cpu_trainer(monkeypatch, attack=[None] * 4 + [("ios_std", 2.0), ("ios_uv", 1.0), None, None], **kw)
    assert tr.byz_pairs == [(4, 0, [0, 1, 3]), (4, 1, [1, 2]), (4, 2, [2, 3]), (4, 7, [7, 0, 1]), (5, 1, [1, 2]),
                            (5, 2, [2, 3]), (5, 3, [3, 0, 1]), (5, 6, [6, 0, 1])]
    assert tr.ios_pairs == list(range(8)) and tr.gamma_pairs == tr.ios_pairs and tr.mom_agents == [2, 6]
    assert all(g == [] for g in tr._attack_job_groups()) and tr._arc_job_groups() == tr._subset_job_groups() == []
    groups = tr._ios_job_groups()
    launches = [(g[0].func, g[0].keywords) if isinstance(g[0], functools.partial) else g[0] for g in groups]
    assert launches == [(ops.ios_history_attack, dict(arc=True)), (ops.ios_pipeline_attack, dict(arc=True)),
                        (ops.ios_pipeline_attack, dict(arc=False)), (ops.subset_history_attack, dict(arc=False)),
                        ops.pipeline_arc_attack]
    assert [(len(g[1]), g[2]) for g in groups] == [(4, [0, 0, 0, 0]), (2, None), (6, None), (2, [1, 1]), (2, None)]
    ios = (L.TAILOR_FILTER, L.FILTER_IOS)
    hist_arc, pipe_arc, pipe_plain, sub_hist, other = (list(g[1]) for g in groups)
    for n, (e, t) in enumerate((e, t) for e in (2, 5) for t in (0, 1)):
        j = hist_arc[n]
        dev, scale = (L.DEV_STD, 2.0) if e == 2 else (L.DEV_UV, 1.0)
        AC._check_base(tr, j, e, t, 2, [2, -1, 3, -1, -1], 0b00101, dev, scale, rule=ios)
        ref = tr.critic[2] if t == 0 else tr.tr[2]
        assert (j.ref, j.momentum, j.momentum_stride) == (ref.data_ptr(), tr.momentum_M[0, t].data_ptr(), tr.PT)
        assert j.beta == f32(0.9) and j.first == 0 and j.own_mask == (0b01010 if e == 2 else 0b10000)
    want = {0: (0, [0, 1, -1, 3], 0b1011, None), 1: (1, [1, 2, -1, -1], 0b0011, "nnm"),
            4: (1, [1, 2, -1, -1], 0b0011, "nnm"), 6: (3, [3, 0, -1, 1], 0b1011, ("bucket", 2))}
    cases = [(pipe_arc, ((0, 0), (0, 1))), (pipe_plain, ((e, t) for e in (1, 4, 6) for t in (0, 1)))]
    for js, pairs in cases:
        for j, (e, t) in zip(js, pairs):
            r, slots, hm, mix = want[e]
            dev, scale = (L.DEV_STD, 2.0) if tr.byz_pairs[e][0] == 4 else (L.DEV_UV, 1.0)
            AC._check_base(tr, j, e, t, r, slots, hm, dev, scale, rule=ios)
            assert j.mixing == (L.PIPE_NONE if mix is None else L.PIPE_NNM if mix == "nnm" else L.PIPE_BUCKET)
            assert j.s == (2 if mix == ("bucket", 2) else 0) and j.n_perms == L.PIPELINE_PERMS
            assert (j.seed, j.attacker, j.receiver, j.net, j.round) == (tr.seed, tr.byz_pairs[e][0], r, t, 0)
    # the same team with subset_* attackers and the ios receivers on clip: its jobs against receivers 6 and 7
    sub = AC._cpu_trainer(monkeypatch, attack=[None] * 4 + [("subset_std", 2.0), ("subset_uv", 1.0), None, None],
                          **dict(kw, aggregation=["clip"] * 4 + agg[4:]))
    sgroups = sub._subset_job_groups()
    (g_hist,) = [g for fn, g, _ in sgroups if isinstance(fn, functools.partial) and fn.func == ops.subset_history_attack]
    (g_arc,) = [g for fn, g, _ in sgroups if fn == ops.pipeline_arc_attack]
    theirs = [j for j in g_arc if j.receiver == 7]
    assert len(sub_hist) == len(g_hist) == len(other) == len(theirs) == 2
    for ja, jb in zip(sub_hist + other, list(g_hist) + theirs):
        assert SC._fields(ja) == SC._fields(jb)


def test_without_an_ios_attacker_no_ios_groups(monkeypatch):
    labels = ["Cooperative"] * 4 + ["Byzantine"]
    tr = AC._cpu_trainer(monkeypatch, labels=labels, in_nodes=C5, desired=np.zeros((5, 2)), aggregation="ios",
                         attack=[None] * 4 + [("gauss", 1.0)])
    assert tr.ios_pairs == [] and tr._ios_job_groups() == []
