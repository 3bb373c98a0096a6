"""CPU checks of the rule-aware attacks (rcmarl_tailored_attack, include/rcmarl.h): properties of the fp64 oracle
(tests/tailored_attack_oracle.py) with hypothesis -- scale 0 sends mu, a plain-mean receiver with only honest real slots
gets the last candidate, at scale 1 the pick does at least the min-max message's damage, and the honest slots' order only
matters through rounding or near ties --, the C layout of the job, and the refusals of the library, the bindings and
Trainer before any device work."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import adaptive_attack_oracle as AA
import attack_oracle as AT
import tailored_attack_oracle as TA
import vector_oracle as VO
from test_attacks_cpu import no_device, trainer   # noqa: F401  (no_device is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f64 = np.float64


def _max_h(rule, n_in):
    return n_in - 3 if rule in ("krum", "mkrum") else ((n_in - 1) // 2 if rule == "trim" else n_in - 1)


@st.composite
def receivers(draw, rules=TA.RULES, malicious=True):
    """(rows, slots, honest, rule, H): a receiver with n_in slots, 1-3 crafted, the real ones honest or far-off rows"""
    rule = draw(st.sampled_from(rules))
    n_in = draw(st.integers(3 if rule in ("krum", "mkrum") else 2, 9))
    n_cr = draw(st.integers(1, min(3, n_in - 1)))
    n_mal = draw(st.integers(0, n_in - 1 - n_cr)) if malicious else 0
    P = draw(st.integers(2, 8))
    seed = draw(st.integers(0, 2 ** 31 - 1))
    rs = np.random.RandomState(seed)
    n_real = n_in - n_cr
    rows = rs.randn(P) + rs.randn(n_real, P) * rs.uniform(0.1, 1, size=(n_real, 1))
    rows[n_real - n_mal:] += 4 * rs.randn(n_mal, P)
    kinds = ["c"] * n_cr + ["r"] * (n_real - 1)
    rs.shuffle(kinds)
    slots, r = [0], 1
    for t in kinds:
        slots.append(-1 if t == "c" else r)
        r += t == "r"
    honest = [k for k, s in enumerate(slots) if 0 <= s < n_real - n_mal]
    H = draw(st.integers(0, _max_h(rule, n_in)))
    return rows, slots, honest, rule, H


@given(receivers(), st.sampled_from(TA.ATTACKS))
@settings(max_examples=60, deadline=None)
def test_scale_zero_gives_mu(rec, attack):
    rows, slots, honest, rule, H = rec
    m, g, O = TA.craft(rows, slots, honest, rule, H, attack, 0.0)
    assert g == 0
    np.testing.assert_array_equal(m, AT.moments(np.stack([rows[slots[k]] for k in honest]))[0])


@given(receivers(rules=("clip",), malicious=False), st.sampled_from(TA.ATTACKS), st.sampled_from([0.5, 1.0, 2.0]))
@settings(max_examples=60, deadline=None)
def test_plain_mean_receiver_with_honest_real_slots_takes_the_last_candidate(rec, attack, s):
    rows, slots, honest, _, _ = rec
    V = np.stack([rows[slots[k]] for k in honest])
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    m, g, O = TA.craft(rows, slots, honest, "clip", 0, attack, s)
    if g_mm > 0 and (d * d).sum() > 0:
        assert (np.diff(O) > 0).all() and g == s * g_mm
        np.testing.assert_allclose(m, AA.craft(V, "minmax_" + attack.split("_")[1], s)[0], rtol=1e-12, atol=1e-12)


@given(receivers(), st.sampled_from(TA.ATTACKS))
@settings(max_examples=60, deadline=None)
def test_at_scale_one_the_pick_does_at_least_the_minmax_damage(rec, attack):
    rows, slots, honest, rule, H = rec
    V = np.stack([rows[slots[k]] for k in honest])
    mm = AA.craft(V, "minmax_" + attack.split("_")[1], 1.0)[0]
    X = np.stack([mm if s < 0 else rows[s] for s in slots])
    o_mm = TA.objective(TA.rule_output(X, rule, H), AT.moments(V)[0])
    m, g, O = TA.craft(rows, slots, honest, rule, H, attack, 1.0)
    assert O.max() >= o_mm * (1 - 1e-9) - 1e-12


@given(receivers(), st.sampled_from(TA.ATTACKS), st.randoms(use_true_random=False))
@settings(max_examples=60, deadline=None)
def test_permuting_the_honest_slots_changes_gamma_only_by_rounding_or_a_near_tie(rec, attack, rnd):
    rows, slots, honest, rule, H = rec
    _, g, O = TA.craft(rows, slots, honest, rule, H, attack, 2.0)
    # permute the rows behind the honest slots other than slot 0 (the receiver's own message stays)
    movable = [k for k in honest if k != 0]
    perm = list(movable)
    rnd.shuffle(perm)
    slots2 = list(slots)
    for a, b in zip(movable, perm):
        slots2[a] = slots[b]
    _, g2, O2 = TA.craft(rows, slots2, honest, rule, H, attack, 2.0)
    if rule in ("krum", "mkrum") and _selection_tie(rows, slots, honest, rule, H, attack):
        return                          # the receiver's own rule breaks an exact score tie by slot index
    if int(np.argmax(O)) != int(np.argmax(O2)):
        # a different pick is only allowed where it is a near tie for both lists
        i2 = int(np.argmax(O2))
        assert O[i2] >= O.max() * (1 - 1e-6) - 1e-12 or TA.margin(O) <= 1e-6
    else:
        np.testing.assert_allclose(g2, g, rtol=1e-9, atol=1e-12)


def _selection_tie(rows, slots, honest, rule, H, attack):
    """True if Krum / multi-Krum meets an exact score tie at its selection boundary for some candidate (at H = n - 3 a
    score is one nearest-neighbour distance, which two mutually nearest messages share): its output then depends on
    the slot order, whatever the attack does."""
    V = np.stack([rows[slots[k]] for k in honest])
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    n = len(slots)
    m = 1 if rule == "krum" else n - H
    for i in range(TA.STEPS + 1):
        c = TA.candidate(mu, d, 2.0 * g_mm * i / TA.STEPS)
        sc = np.sort(VO.krum_scores(np.stack([c if s < 0 else rows[s] for s in slots]), H))
        if m < n and sc[m - 1] == sc[m]:
            return True
    return False


def test_a_range_beyond_fp32_gives_mu():
    rows = np.array([[0.0, 0.0], [8.0, 1.0], [-8.0, 3.0], [1.0, -9.0]])
    slots, honest = [0, 1, 2, 3, -1], [0, 1, 2, 3]
    m, g, O = TA.craft(rows, slots, honest, "clip", 0, "tailored_std", 3e38)
    assert g == 0 and (O == 0).all()
    np.testing.assert_array_equal(m, rows.mean(0))


def test_ties_go_to_the_smaller_index():
    """A trimmed-mean receiver that drops the crafted slot for every gamma > 0: O is flat from i = 1 on, i* = 1."""
    rows = np.array([[0.0, 0.0], [1.0, 0.0], [-1.0, 0.0], [0.0, 1.0]])
    slots, honest = [0, 1, 2, 3, -1], [0, 1, 2, 3]
    m, g, O = TA.craft(rows, slots, honest, "trim", 1, "tailored_uv", 2.0)
    assert np.isfinite(O).all()
    i = int(np.argmax(O))
    assert (O[i:] == O[i]).sum() >= 2 and g == TA.craft(rows, slots, honest, "trim", 1, "tailored_uv", 2.0)[1]
    assert i == min(np.flatnonzero(O == O.max()))


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_tailored_attack_job_layout_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = ["dst", "msgs", "msg_stride", "gamma_out", "n", "n_in", "slots", "honest_mask", "family", "rule", "H",
              "dev", "scale"]
    enums = ["RCMARL_TAILOR_COORD", "RCMARL_TAILOR_VECTOR", "RCMARL_TAILORED_STEPS", "RCMARL_TAILORED_MAX_FLOATS"]
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'printf("%zu", sizeof(rcmarl_tailored_attack_job));'
                   + "".join(f'printf(" %zu", offsetof(rcmarl_tailored_attack_job, {f}));' for f in fields)
                   + "".join(f'printf(" %d", (int)({e}));' for e in enums) + 'printf("\\n"); return 0;}')
    exe = tmp_path / "off"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == ctypes.sizeof(L.TailoredAttackJob) == 128
    assert got[1:1 + len(fields)] == [getattr(L.TailoredAttackJob, f).offset for f in fields]
    assert got[1 + len(fields):] == [L.TAILOR_COORD, L.TAILOR_VECTOR, L.TAILORED_STEPS, L.TAILORED_MAX_FLOATS] \
        == [0, 1, TA.STEPS, 19 * 1536]
    assert ("rcmarl_tailored_attack", ctypes.c_int, [ctypes.POINTER(L.TailoredAttackJob), ctypes.c_int, L.c_fp]) \
        in L.SYMBOLS


P_FAKE, STRIDE = 100, 128                       # fake device addresses: rows of msgs at 1 MiB + r * 512 bytes
MSGS = 1 << 20
ROW5 = MSGS + 5 * STRIDE * 4


def _job(**kw):
    from rcmarl import _lib as L
    j = L.TailoredAttackJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in = 1 << 24, MSGS, STRIDE, P_FAKE, 3
    j.family, j.rule, j.H, j.dev, j.scale = L.TAILOR_COORD, L.AGG_CLIP, 0, L.DEV_STD, 2.0
    j.slots[0], j.slots[1], j.slots[2] = 0, -1, 1
    j.honest_mask = 0b101
    for k, v in kw.items():
        if k == "slots":
            for i, x in enumerate(v):
                j.slots[i] = x
        else:
            setattr(j, k, v)
    return j


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-3), dict(n_in=0), dict(n_in=17),
    dict(slots=[0, 2, 1]),                                             # no crafted slot
    dict(honest_mask=0),                                               # no honest slot
    dict(honest_mask=0b111),                                           # a crafted slot marked honest
    dict(honest_mask=0b1001),                                          # a bit past n_in
    dict(slots=[0, -2, 1]),                                            # a slot below -1
    dict(family=2), dict(family=-1), dict(rule=3), dict(family=1, rule=4), dict(family=1, rule=-1),
    dict(dev=3), dict(dev=-1), dict(H=-1), dict(H=3),
    dict(rule=1, H=2),                                                 # trim: 2H >= n_in
    dict(family=1, rule=0, H=1, n_in=3),                               # krum: n_in < H + 3
    dict(family=1, rule=1, n_in=2, slots=[0, -1]),                     # mkrum: n_in < H + 3
    dict(scale=float("nan")), dict(scale=float("inf")), dict(scale=-0.5),
    dict(n=19 * 1536 // 6 + 1, msg_stride=8192),                       # (3 + 3) * n over the staging bound
    dict(dst=MSGS + STRIDE * 4 - 8),                                   # dst overlaps real slot row 0 (of this job)
    dict(dst=ROW5 + 40),                                               # ... a real slot of the other job
    dict(gamma_out=MSGS + STRIDE * 4 + 12),                            # gamma_out on one of its real rows
    dict(gamma_out=ROW5 + 4 * 8),                                      # ... on the other job's real row
    dict(gamma_out=(1 << 25) + 4),                                     # ... on the other job's dst
    dict(gamma_out=1 << 26),                                           # ... on the other job's gamma_out
    dict(dst=(1 << 25) + 4 * (P_FAKE - 1)),                            # two dsts overlap
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    good = _job(dst=1 << 25, gamma_out=1 << 26, slots=[5, -1, 6])
    for jobs in ([good, _job(**bad)], [_job(**bad), good]):
        arr = (L.TailoredAttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_tailored_attack(arr, len(arr), None) == -1           # RCMARL_ERR_ARG


def test_library_refuses_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_tailored_attack(None, 1, None) == -1
    arr = (L.TailoredAttackJob * 33)(*[_job(dst=(1 << 24) + (1 << 12) * i) for i in range(33)])
    assert lib.rcmarl_tailored_attack(arr, 0, None) == -1
    assert lib.rcmarl_tailored_attack(arr, 33, None) == -1


def test_staging_bound_is_the_trainers_largest_job():
    from rcmarl import _lib as L
    assert (16 + 3) * L.param_count(48, 1) <= L.TAILORED_MAX_FLOATS < (16 + 3) * 1537
    assert 4 * L.TAILORED_MAX_FLOATS + 1376 <= 227 * 1024          # with the kernel's static shared memory, per CTA


def test_attack_names_and_parameters():
    from rcmarl import _lib as L
    for name in TA.ATTACKS:
        kind, s = L.check_attack((name, 2))
        assert kind == L.TAILORED_ATTACKS[name] and isinstance(kind, L.TailoredKind) and s == 2.0
        assert not isinstance(kind, tuple) and L.is_tailored_attack(name) and not L.is_adaptive_attack(name)
        for bad in [(name, -1e-3), (name, float("nan")), (name, float("inf")), (name, "x"), (name,)]:
            with pytest.raises(L.RcmarlError):
                L.check_attack(bad)
    assert [int(L.TAILORED_ATTACKS[a]) for a in TA.ATTACKS] == [L.DEV_UV, L.DEV_STD, L.DEV_SGN]
    assert L.check_attack(("alie", -2)) == (0, -2.0) and L.check_attack(("minmax_std", 1)) == ((0, 1), 1.0)
    for bad in [("tailored", 1), ("tailored_l2", 1), ("TAILORED_UV", 1)]:
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)


def test_bindings_refuse_unknown_names_and_fill_the_job():
    import torch
    from rcmarl import _lib as L, ops
    x = torch.zeros(4, 8)
    with pytest.raises(L.RcmarlError):
        ops.tailored_attack_job(x[3], x, 8, 8, [0, -1], [0], "clip", 0, "tailored", 1.0)
    with pytest.raises(L.RcmarlError):
        ops.tailored_attack_job(x[3], x, 8, 8, [0, -1], [0], "clip", 0, "minmax_uv", 1.0)
    with pytest.raises(L.RcmarlError):
        ops.tailored_attack_job(x[3], x, 8, 8, [0, -1], [0], "median", 0, "tailored_uv", 1.0)
    for honest in ([0, 2], [0, -1], [0, 32], [0, 1.0]):                     # outside the 2 slots, or not an index
        with pytest.raises(L.RcmarlError):
            ops.tailored_attack_job(x[3], x, 8, 8, [0, -1], honest, "clip", 0, "tailored_uv", 1.0)
    j = ops.tailored_attack_job(x[3], x, 8, 8, [0, -1, 2, 1], [0, 3], "gmed", 1, "tailored_sgn", 0.5,
                                gamma_out=x[3, :1])
    assert (j.n_in, list(j.slots)[:4], j.honest_mask, j.family, j.rule, j.H, j.dev, j.scale) == \
        (4, [0, -1, 2, 1], 0b1001, L.TAILOR_VECTOR, L.VEC_GMED, 1, L.DEV_SGN, 0.5)
    j = ops.tailored_attack_job(x[3], x, 8, 8, [0, -1], [0], "wmsr", 0, "tailored_uv", 2.0)
    assert (j.family, j.rule, j.gamma_out) == (L.TAILOR_COORD, L.AGG_WMSR, None)


@pytest.mark.parametrize("attack", [("tailored_std", -1.0), ("tailored_uv", float("nan")), ("tailored", 1.0),
                                    [None] * 4 + [("tailored_sgn", float("inf"))]])
def test_trainer_refuses_invalid_tailored_attacks_before_any_device_work(no_device, attack):   # noqa: F811
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(attack, H=0)


@pytest.mark.parametrize("attack,labels", [
    (("tailored_std", 2.0), None),
    ([None] * 4 + [("tailored_uv", 0.0)], None),
    ([("tailored_sgn", 2.0), None, ("minmax_std", 1.0), None, None], ["Byzantine", "Cooperative", "Byzantine",
                                                                      "Cooperative", "Cooperative"]),
])
def test_trainer_accepts_tailored_attacks(no_device, attack, labels):   # noqa: F811
    with pytest.raises(no_device):
        trainer(attack, labels)
