"""CPU checks of the dissensus and mimic attacks (rcmarl_dissensus_attack, rcmarl_mimic_attack, include/rcmarl.h):
properties of the oracle (tests/dissensus_mimic_oracle.py) with hypothesis -- eps = 0 sends x, one attacker at eps = 1
leaves a plain-mean receiver at x, the message is linear in eps; the mimic message is a candidate row, its choice is
equivariant under a permutation of S_j, one power step on a rank-1 spread gives +-its direction, and fp32 agrees with
fp64 --, hand-worked examples, the C layout of the jobs, and the refusals of the library, the bindings and Trainer
before any device work."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dissensus_mimic_oracle as DM
from test_attacks_cpu import no_device, trainer   # noqa: F401  (no_device is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f64 = np.float64


@st.composite
def honest_sets(draw, n_min=1):
    """(x, V): the receiver's own message and n honest rows around a common centre (x among them), P small."""
    n = draw(st.integers(n_min, 16))
    P = draw(st.integers(1, 12))
    rs = np.random.RandomState(draw(st.integers(0, 2 ** 31 - 1)))
    V = rs.randn(P) + rs.randn(n, P) * rs.uniform(0.1, 2, size=(n, 1))
    if n >= 3 and draw(st.booleans()):
        V[-1] = V[0]                                     # a repeated entry
    return V[0].copy(), V


# ------------------------------------------------------------------------------------------------ dissensus
@given(honest_sets(), st.integers(1, 16))
@settings(max_examples=80, deadline=None)
def test_dissensus_eps_zero_sends_x_bitwise(xv, n_byz):
    x, V = xv
    for dt in (np.float32, f64):
        np.testing.assert_array_equal(DM.dissensus(x.astype(dt), V.astype(dt), n_byz, 0.0), x.astype(dt))


@given(honest_sets())
@settings(max_examples=80, deadline=None)
def test_one_attacker_at_eps_one_leaves_a_plain_mean_receiver_at_x(xv):
    """A receiver that averages its n honest messages (itself among them) and one dissensus message stays at x."""
    x, V = xv
    m = DM.dissensus(x, V, 1, 1.0)
    mean = (V.sum(0) + m) / (len(V) + 1)
    np.testing.assert_allclose(mean, x, rtol=0, atol=1e-12 * (1 + np.abs(V).max()) * len(V))


@given(honest_sets(), st.integers(1, 16), st.floats(0, 8), st.floats(0, 8))
@settings(max_examples=80, deadline=None)
def test_dissensus_is_linear_in_eps(xv, n_byz, a, b):
    x, V = xv
    ma, mb, mab = (DM.dissensus(x, V, n_byz, e) for e in (a, b, a + b))
    np.testing.assert_allclose(mab - x, (ma - x) + (mb - x), rtol=1e-9, atol=1e-9 * (1 + np.abs(V).max()) * len(V))


@given(honest_sets(), st.integers(1, 16), st.floats(0, 4))
@settings(max_examples=60, deadline=None)
def test_dissensus_fp32_agrees_with_fp64(xv, n_byz, eps):
    x, V = xv
    x32, V32 = x.astype(np.float32), V.astype(np.float32)
    got = DM.dissensus(x32, V32, n_byz, eps)
    want = DM.dissensus(x32.astype(f64), V32.astype(f64), n_byz, eps)
    np.testing.assert_allclose(got, want, rtol=0, atol=4e-7 * (1 + eps) * len(V) * (1 + np.abs(V32).max()))


def test_dissensus_by_hand():
    """x = (1, 0), honest rows x, (3, 0), (1, 4): delta = (2, 4); two attackers at eps = 1 send x - delta / 2."""
    x = np.array([1.0, 0.0])
    V = np.array([[1.0, 0.0], [3.0, 0.0], [1.0, 4.0]])
    np.testing.assert_array_equal(DM.dissensus(x, V, 2, 1.0), [0.0, -2.0])
    np.testing.assert_array_equal(DM.dissensus(x, V, 1, 3.0), [-5.0, -12.0])


# ------------------------------------------------------------------------------------------------ mimic
@st.composite
def mimic_cases(draw):
    _, V = draw(honest_sets())
    n = len(V)
    cand = sorted(draw(st.sets(st.integers(0, n - 1), min_size=1)))
    rs = np.random.RandomState(draw(st.integers(0, 2 ** 31 - 1)))
    z = np.zeros(V.shape[1]) if draw(st.booleans()) else rs.randn(V.shape[1])
    return V, cand, z, draw(st.sampled_from([0, 1]))


@given(mimic_cases())
@settings(max_examples=100, deadline=None)
def test_mimic_sends_a_candidate_row(case):
    V, cand, z, update = case
    k, z2, t = DM.mimic(V, cand, z, update)
    assert k in cand
    if update == 0 and z.any():
        np.testing.assert_array_equal(z2, z)
    if z2.any() and not z.any():                         # set by Init (and perhaps a step): a unit vector
        np.testing.assert_allclose(np.linalg.norm(z2), 1.0, rtol=1e-12)


@given(mimic_cases(), st.randoms(use_true_random=False))
@settings(max_examples=100, deadline=None)
def test_mimic_choice_is_equivariant_under_a_permutation_of_the_honest_set(case, rnd):
    """Permuting S_j (and the candidate set with it) copies the same row, unless the pick or the Init is a near tie."""
    V, cand, z, update = case
    perm = list(range(len(V)))
    rnd.shuffle(perm)                                    # new entry i is old entry perm[i]
    inv = {o: i for i, o in enumerate(perm)}
    k, z1, t = DM.mimic(V, cand, z, update)
    k2, z2, t2 = DM.mimic(V[perm], [inv[c] for c in cand], z, update)
    if DM.init_margin(V) < 1e-9 and not z.any():
        return                                           # the Init picks the first of equal rows: index dependent
    if DM.pick_margin(V, t) > 1e-9:
        np.testing.assert_array_equal(V[perm][k2], V[k])
    np.testing.assert_allclose(z2, z1, rtol=1e-9, atol=1e-12)


@given(st.integers(2, 16), st.integers(2, 12), st.integers(0, 2 ** 31 - 1), st.booleans())
@settings(max_examples=80, deadline=None)
def test_one_power_step_on_a_rank_one_spread_gives_its_direction(n, P, seed, from_init):
    """Honest rows mu0 + a_k d: after one step from any z not orthogonal to d, z = +-d / ||d||."""
    rs = np.random.RandomState(seed)
    d = rs.randn(P)
    a = rs.randn(n)
    V = rs.randn(P) + np.outer(a, d)
    z = np.zeros(P) if from_init else rs.randn(P)
    if abs(z @ d) < 1e-3 * np.linalg.norm(z) * np.linalg.norm(d) and not from_init:
        return
    _, z2, _ = DM.mimic(V, range(n), z, 1)
    np.testing.assert_allclose(abs(z2 @ d) / np.linalg.norm(d), 1.0, rtol=1e-9)


@given(mimic_cases())
@settings(max_examples=100, deadline=None)
def test_mimic_fp32_agrees_with_fp64(case):
    V, cand, z, update = case
    V32, z32 = V.astype(np.float32), z.astype(np.float32)
    k64, z64, t64 = DM.mimic(V32.astype(f64), cand, z32.astype(f64), update)
    if not z32.any() and DM.init_margin(V32.astype(f64)) < 1e-4:
        return
    k32, zz, t32 = DM.mimic(V32, cand, z32, update)
    if z64.any():
        assert abs(float(zz.astype(f64) @ z64) / np.linalg.norm(z64) / max(np.linalg.norm(zz), 1e-30)) > 1 - 1e-4
    if DM.pick_margin(V32.astype(f64), t64) > 1e-4:
        np.testing.assert_array_equal(V32[k32], V32[k64])


def test_mimic_by_hand():
    """Rows (0, 0), (2, 0), (4, 1): mu = (2, 1/3), centred (-2, -1/3), (0, -1/3), (2, 2/3); Init takes row 2 (e =
    4 + 4/9), z = (2, 2/3) / sqrt(40/9); the step keeps the larger spread along x; the candidate furthest along z is row
    2, and without it row 1 (t_1 = -2/9 / ... > t_0)."""
    V = np.array([[0.0, 0.0], [2.0, 0.0], [4.0, 1.0]])
    k, z, t = DM.mimic(V, [0, 1, 2], np.zeros(2), 0)
    np.testing.assert_allclose(z, np.array([2.0, 2 / 3]) / np.sqrt(40 / 9), rtol=1e-15)
    assert k == 2
    k, z, t = DM.mimic(V, [0, 1], np.zeros(2), 0)
    assert k == 1
    C = V - V.mean(0)
    k, z1, _ = DM.mimic(V, [0, 1], np.zeros(2), 1)
    u = C.T @ (C @ (C[2] / np.linalg.norm(C[2])))
    np.testing.assert_allclose(z1, u / np.linalg.norm(u), rtol=1e-14)
    # equal rows: z stays 0 and the lowest candidate is copied
    k, z, t = DM.mimic(np.ones((3, 4)), [2, 1], np.zeros(4), 1)
    assert k == 1 and not z.any()
    # an S_j of the receiver alone
    k, z, t = DM.mimic(np.ones((1, 4)) * 3, [0], np.zeros(4), 1)
    assert k == 0 and not z.any()


def test_candidates_drop_the_receiver_unless_none_remain():
    assert DM.candidates(2, [2, 3, 0, 2]) == [1, 2]
    assert DM.candidates(2, [2, 2]) == [0, 1]


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def _layout(tmp_path, struct, fields, enums):
    src = tmp_path / f"{struct}.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   f'printf("%zu", sizeof({struct}));'
                   + "".join(f'printf(" %zu", offsetof({struct}, {f}));' for f in fields)
                   + "".join(f'printf(" %d", (int)({e}));' for e in enums) + 'printf("\\n"); return 0;}')
    exe = tmp_path / struct
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return [int(x) for x in subprocess.check_output([str(exe)]).split()]


def test_job_layouts_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = ["dst", "msgs", "msg_stride", "n", "own", "n_honest", "honest", "n_byz", "eps", "reserved"]
    got = _layout(tmp_path, "rcmarl_dissensus_job", fields, [])
    assert got[0] == ctypes.sizeof(L.DissensusJob) == 112
    assert got[1:] == [getattr(L.DissensusJob, f).offset for f in fields]
    fields = ["dst", "msgs", "msg_stride", "z", "target_out", "n", "n_honest", "honest", "candidate_mask", "update"]
    got = _layout(tmp_path, "rcmarl_mimic_job", fields, ["RCMARL_MIMIC_MAX_FLOATS"])
    assert got[0] == ctypes.sizeof(L.MimicJob) == 120
    assert got[1:-1] == [getattr(L.MimicJob, f).offset for f in fields]
    assert got[-1] == L.MIMIC_MAX_FLOATS == 19 * 1536
    assert ("rcmarl_dissensus_attack", ctypes.c_int, [ctypes.POINTER(L.DissensusJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert ("rcmarl_mimic_attack", ctypes.c_int, [ctypes.POINTER(L.MimicJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS


P_FAKE, STRIDE = 100, 128                       # fake device addresses: rows of msgs at 1 MiB + r * 512 bytes
MSGS = 1 << 20
ROW5 = MSGS + 5 * STRIDE * 4


def _djob(**kw):
    from rcmarl import _lib as L
    j = L.DissensusJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.own, j.n_honest, j.n_byz, j.eps = 1 << 24, MSGS, STRIDE, P_FAKE, 0, 2, 1, 1.0
    j.honest[0], j.honest[1] = 0, 1
    for k, v in kw.items():
        if k == "honest":
            for i, x in enumerate(v):
                j.honest[i] = x
        else:
            setattr(j, k, v)
    return j


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-3), dict(n_honest=0), dict(n_honest=17),
    dict(honest=[0, -1]), dict(own=-1), dict(n_byz=0), dict(n_byz=17),
    dict(eps=float("nan")), dict(eps=float("inf")), dict(eps=-0.5),
    dict(dst=MSGS + STRIDE * 4 - 8),                                   # dst overlaps honest row 0 of this job
    dict(dst=MSGS + 3 * STRIDE * 4, own=3),                            # ... its own row
    dict(dst=ROW5 + 40),                                               # ... an honest row of the other job
    dict(dst=MSGS + 7 * STRIDE * 4 + 4),                               # ... the other job's own row
    dict(dst=(1 << 25) + 4 * (P_FAKE - 1)),                            # two dsts overlap
])
def test_dissensus_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    good = _djob(dst=1 << 25, honest=[5, 6], own=7)
    for jobs in ([good, _djob(**bad)], [_djob(**bad), good]):
        arr = (L.DissensusJob * len(jobs))(*jobs)
        assert lib.rcmarl_dissensus_attack(arr, len(arr), None) == -1           # RCMARL_ERR_ARG


def _mjob(**kw):
    from rcmarl import _lib as L
    j = L.MimicJob()
    j.dst, j.msgs, j.msg_stride, j.z, j.n, j.n_honest = 1 << 24, MSGS, STRIDE, (1 << 24) + 4096, P_FAKE, 3
    j.honest[0], j.honest[1], j.honest[2] = 0, 1, 2
    j.candidate_mask, j.update = 0b110, 1
    for k, v in kw.items():
        if k == "honest":
            for i, x in enumerate(v):
                j.honest[i] = x
        else:
            setattr(j, k, v)
    return j


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(z=None), dict(n=0), dict(n=-3), dict(n_honest=0), dict(n_honest=17),
    dict(honest=[0, -1, 2]), dict(candidate_mask=0), dict(candidate_mask=0b1010),   # a bit at n_honest
    dict(candidate_mask=1 << 31), dict(update=2), dict(update=-1),
    dict(n=19 * 1536 // 6 + 1, msg_stride=8192),                       # (3 + 3) * n over the staging bound
    dict(dst=MSGS + STRIDE * 4 - 8),                                   # dst overlaps honest row 0 of this job
    dict(dst=ROW5 + 40),                                               # ... an honest row of the other job
    dict(z=MSGS + 2 * STRIDE * 4 + 12),                                # z on one of its honest rows
    dict(z=ROW5 + 4 * 8),                                              # ... on the other job's honest row
    dict(z=(1 << 25) + 4),                                             # ... on the other job's dst
    dict(z=1 << 24, dst=(1 << 24) + 200),                              # its own dst and z overlap
    dict(target_out=MSGS + 4),                                         # target_out on an honest row
    dict(target_out=(1 << 26) + 8),                                    # ... on the other job's z
    dict(target_out=1 << 27),                                          # ... on the other job's target_out
    dict(dst=(1 << 25) + 4 * (P_FAKE - 1)),                            # two dsts overlap
])
def test_mimic_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    good = _mjob(dst=1 << 25, z=1 << 26, target_out=1 << 27, honest=[5, 6, 7])
    for jobs in ([good, _mjob(**bad)], [_mjob(**bad), good]):
        arr = (L.MimicJob * len(jobs))(*jobs)
        assert lib.rcmarl_mimic_attack(arr, len(arr), None) == -1


def test_library_refuses_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_dissensus_attack(None, 1, None) == -1
    assert lib.rcmarl_mimic_attack(None, 1, None) == -1
    d = (L.DissensusJob * 33)(*[_djob(dst=(1 << 24) + (1 << 12) * i) for i in range(33)])
    m = (L.MimicJob * 33)(*[_mjob(dst=(1 << 24) + (1 << 13) * i, z=(1 << 24) + (1 << 13) * i + 4096) for i in range(33)])
    for f, arr in ((lib.rcmarl_dissensus_attack, d), (lib.rcmarl_mimic_attack, m)):
        assert f(arr, 0, None) == -1 and f(arr, 33, None) == -1


def test_staging_bound_is_the_trainers_largest_job():
    from rcmarl import _lib as L
    assert (16 + 3) * L.param_count(48, 1) <= L.MIMIC_MAX_FLOATS < (16 + 3) * 1537
    assert 4 * L.MIMIC_MAX_FLOATS + 80 <= 227 * 1024              # with the kernel's static shared memory, per CTA


def test_attack_names_and_parameters():
    from rcmarl import _lib as L
    kind, eps = L.check_attack(("dissensus", 1))
    assert isinstance(kind, L.DissensusKind) and eps == 1.0 and not isinstance(kind, (tuple, L.TailoredKind))
    kind, t0 = L.check_attack(("mimic", 50))
    assert isinstance(kind, L.MimicKind) and t0 == 50.0 and not isinstance(kind, (tuple, L.TailoredKind))
    assert L.check_attack(("dissensus", 0))[1] == 0.0 and L.check_attack(("mimic", 0))[1] == 0.0
    assert L.check_attack(("mimic", 2 ** 31 - 1))[1] == 2 ** 31 - 1 and L.check_attack(("mimic", 7.0))[1] == 7.0
    for bad in [("dissensus", -1e-3), ("dissensus", float("nan")), ("dissensus", float("inf")), ("dissensus", "x"),
                ("mimic", 1.5), ("mimic", -1), ("mimic", 2 ** 31), ("mimic", float("inf")), ("mimic", float("nan")),
                ("mimic",), ("Mimic", 1), ("dissent", 1)]:
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)
    assert L.check_attack(("alie", -2)) == (0, -2.0) and L.check_attack(("minmax_std", 1)) == ((0, 1), 1.0)


def test_bindings_fill_the_jobs():
    import torch
    from rcmarl import _lib as L, ops
    x = torch.zeros(6, 8)
    z = torch.zeros(8)
    for cand in ([3], [-1], [0, 1.0]):
        with pytest.raises(L.RcmarlError):
            ops.mimic_attack_job(x[5], x, 8, 8, [0, 1, 2], cand, z, 1)
    j = ops.mimic_attack_job(x[5], x, 8, 8, [2, 0, 1], [2, 0], z, 1, target_out=None)
    assert (j.n_honest, list(j.honest)[:3], j.candidate_mask, j.update, j.target_out) == (3, [2, 0, 1], 0b101, 1, None)
    j = ops.dissensus_attack_job(x[5], x, 8, 8, 2, [2, 0, 2], 3, 1.5)
    assert (j.own, j.n_honest, list(j.honest)[:3], j.n_byz, j.eps) == (2, 3, [2, 0, 2], 3, 1.5)


# ------------------------------------------------------------------------------------------------ Trainer
@pytest.mark.parametrize("attack", [("dissensus", -1.0), ("dissensus", float("nan")), ("mimic", 0.5), ("mimic", -2),
                                    ("mimic", 2 ** 31), [None] * 4 + [("mimic", float("inf"))]])
def test_trainer_refuses_invalid_attacks_before_any_device_work(no_device, attack):   # noqa: F811
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(attack, H=0)


def _pairs_without_device(monkeypatch, attack, labels=None, in_nodes=None, aggregation="clip", mixing=None):
    """Trainer.__init__ up to its first device allocation: the pair lists and the message-row count it would use."""
    import torch
    from rcmarl.trainer import Trainer
    from test_attacks_cpu import C5
    seen = {}

    class Stop(Exception):
        pass

    def zeros(*a, **k):
        seen.setdefault("shape", a)
        raise Stop()
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch, "zeros", zeros)
    labels = labels or ["Cooperative"] * 4 + ["Byzantine"]
    tr = Trainer.__new__(Trainer)
    with pytest.raises(Stop):
        tr.__init__(labels=labels, in_nodes=in_nodes or C5, weights=[], desired=np.zeros((len(labels), 2)), H=1,
                    aggregation=aggregation, attack=attack, mixing=mixing)
    return tr


def test_trainer_pair_lists_and_rows(monkeypatch):
    labels = ["Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative"]
    in_nodes = [[0, 1, 2, 3], [1, 0], [2, 1, 3, 4], [3, 2], [4, 5, 5, 6], [5, 4], [6, 1, 5, 0]]
    att = [None, ("dissensus", 1.0), None, ("mimic", 5), None, ("alie", 1.0), None]
    tr = _pairs_without_device(monkeypatch, att, labels, in_nodes)
    assert [p[:2] for p in tr.byz_pairs] == [(1, 0), (1, 2), (1, 6), (3, 0), (3, 2), (5, 4), (5, 6)]
    assert tr.diss_pairs == [0, 1, 2] and tr.mimic_pairs == [3, 4]
    assert tr.adapt_pairs == tr.tailor_pairs == [] and tr.gamma_pairs == []
    # the message rows: one per agent slot and one per pair, as for every other attack
    tr2 = _pairs_without_device(monkeypatch, [None, ("alie", 1.0), None, ("ipm", 1.0), None, ("alie", 1.0), None],
                                labels, in_nodes)
    assert len(tr.byz_pairs) == len(tr2.byz_pairs)
    assert tr.vec_row == tr2.vec_row and tr.dnc_row == tr2.dnc_row and tr.mix_row == tr2.mix_row


@pytest.mark.parametrize("aggregation,mixing", [("dnc", None), ("clip", "nnm"), ("krum", "nnm"), ("scclip", None)])
def test_the_new_attacks_are_refused_by_no_rule_and_no_mixing(monkeypatch, aggregation, mixing):
    from test_attacks_cpu import C5
    for att in (("dissensus", 2.0), ("mimic", 3)):
        in_nodes = [list(x) + [x[0]] * 2 if aggregation == "krum" else x for x in C5]
        tr = _pairs_without_device(monkeypatch, att, in_nodes=in_nodes, aggregation=aggregation, mixing=mixing)
        assert len(tr.diss_pairs if att[0] == "dissensus" else tr.mimic_pairs) == 3


def test_state_dict_keys_only_with_a_mimic_pair():
    """state_dict gains mimic_z / mimic_steps only when a mimic pair exists; loading refuses a checkpoint without them
    or with other shapes (checked before anything is copied)."""
    import torch
    from rcmarl import _lib as L
    from rcmarl.trainer import Trainer
    base = dict(labels=["Cooperative", "Byzantine"], n_envs=1, t_filled=0, episodes_done=0, adam_t=[0, 0])

    class Fake:
        mimic_pairs = []
        labels = base["labels"]
        N = 1
        t_filled = episodes_done = 0
        adam_t = [0, 0]
        _perm_gen = torch.Generator()
        actor = critic = tr = critic_local = adam_m = adam_v = sa = ns = r = torch.zeros(1, 1)
    f = Fake()
    assert "mimic_z" not in Trainer.state_dict(f) and "mimic_steps" not in Trainer.state_dict(f)
    f.mimic_pairs, f.mimic_z, f.mimic_steps = [0], torch.zeros(1, 2, 4), [3]
    sd = Trainer.state_dict(f)
    assert sd["mimic_steps"] == [3] and tuple(sd["mimic_z"].shape) == (1, 2, 4)
    for drop in ("mimic_z", "mimic_steps"):
        with pytest.raises(L.RcmarlError):
            Trainer.load_state_dict(f, {k: v for k, v in sd.items() if k != drop})
    with pytest.raises(L.RcmarlError):
        Trainer.load_state_dict(f, dict(sd, mimic_z=torch.zeros(1, 2, 5)))
    with pytest.raises(L.RcmarlError):
        Trainer.load_state_dict(f, dict(sd, mimic_steps=[1, 2]))
