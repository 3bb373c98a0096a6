"""CPU checks of the selectable resilient aggregation rules (rcmarl_agg_rule, include/rcmarl.h): properties of the
oracle's trim / W-MSR means (tests/agg_oracle.py), the oracle against a direct sort-based restatement, the C layout of
the new job field, and the Trainer's refusal of an invalid rule or H before it touches a device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import agg_oracle as AO
from oracle import rpbcac_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULES = ("trim", "wmsr")
HONEST = st.floats(-1e3, 1e3, allow_nan=False, width=64)
BYZANTINE = st.one_of(st.sampled_from([np.inf, -np.inf, 1e30, -1e30, 1e8, -1e8]),
                      st.floats(allow_nan=False, allow_infinity=True, width=64))


@st.composite
def columns(draw, min_n=1):
    """(values [n, P] float64, H) with ties likely: P columns drawn from a small pool."""
    n = draw(st.integers(min_n, 16))
    P = draw(st.integers(1, 4))
    pool = draw(st.lists(HONEST, min_size=1, max_size=6))
    v = np.array(draw(st.lists(st.sampled_from(pool) | HONEST, min_size=n * P, max_size=n * P)), np.float64)
    return v.reshape(n, P)


def max_H(rule, n):
    return (n - 1) // 2 if rule == "trim" else n - 1


@given(columns(), st.sampled_from(RULES))
@settings(max_examples=200, deadline=None)
def test_H0_is_the_mean(v, rule):
    np.testing.assert_allclose(AO.resilient_aggregation(v, 0, rule), v.mean(0), rtol=1e-12, atol=1e-12)


@given(columns())
@settings(max_examples=200, deadline=None)
def test_trim_at_the_largest_H_is_the_median(v):
    H = (v.shape[0] - 1) // 2
    np.testing.assert_allclose(AO.resilient_aggregation(v, H, "trim"), np.median(v, axis=0), rtol=1e-12, atol=1e-12)


@given(columns(), st.data())
@settings(max_examples=200, deadline=None)
def test_wmsr_keeps_own_and_every_value_equal_to_it(v, data):
    H = data.draw(st.integers(0, v.shape[0] - 1))
    keep = AO.keep_mask(v, H, "wmsr")
    assert keep[0].all()
    assert keep[v == v[0]].all()
    # at most H dropped on each side of own, and only strictly above / below it
    above, below = v > v[0], v < v[0]
    assert ((~keep) & ~(above | below)).sum() == 0
    assert ((~keep) & above).sum(0).max() <= H and ((~keep) & below).sum(0).max() <= H


@given(columns(min_n=2), st.sampled_from(RULES), st.data())
@settings(max_examples=200, deadline=None)
def test_invariant_to_permuting_the_neighbours(v, rule, data):
    H = data.draw(st.integers(0, max_H(rule, v.shape[0])))
    p = data.draw(st.permutations(range(1, v.shape[0])))
    w = v[[0] + list(p)]
    np.testing.assert_allclose(AO.resilient_aggregation(w, H, rule), AO.resilient_aggregation(v, H, rule),
                               rtol=1e-12, atol=1e-9)


@given(st.sampled_from(RULES), st.data())
@settings(max_examples=300, deadline=None)
def test_at_most_H_byzantine_values_stay_within_the_honest_range(rule, data):
    n = data.draw(st.integers(1, 16))
    H = data.draw(st.integers(0, max_H(rule, n)))
    n_bad = data.draw(st.integers(0, min(H, n - 1)))             # own (v[0]) is honest
    v = np.array(data.draw(st.lists(HONEST, min_size=n, max_size=n)), np.float64)
    bad = data.draw(st.lists(st.sampled_from(range(1, n)), min_size=n_bad, max_size=n_bad, unique=True)) if n > 1 else []
    for k in bad:
        v[k] = data.draw(BYZANTINE)
    honest = np.delete(v, bad)
    got = float(AO.resilient_aggregation(v[:, None], H, rule)[0])
    tol = 1e-12 * max(1.0, np.abs(honest).max())
    assert honest.min() - tol <= got <= honest.max() + tol, (v, H, rule, got)


def restated(col, H, rule):
    """The rule as its definition reads, one column at a time with Python lists."""
    own, n = col[0], len(col)
    if rule == "trim":
        kept = sorted(col)[H:n - H]
    else:
        above = sorted(x for x in col if x > own)
        below = sorted(x for x in col if x < own)
        kept = below[min(H, len(below)):] + [x for x in col if x == own] + above[:len(above) - min(H, len(above))]
    return sum(kept) / len(kept)


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("n", range(1, 17))
def test_against_a_sort_based_restatement_with_ties(rule, n):
    rs = np.random.RandomState(100 + n)
    P = 64
    v = rs.randint(-3, 4, size=(n, P)).astype(np.float64)              # many ties, including with own
    v[:, :8] = rs.randn(n, 8)                                          # and some without
    for H in range(max_H(rule, n) + 1):
        got = AO.resilient_aggregation(v, H, rule)
        want = [restated(list(v[:, p]), H, rule) for p in range(P)]
        np.testing.assert_allclose(got, want, rtol=1e-14, atol=1e-14, err_msg=f"{rule} n={n} H={H}")


def test_fp32_matches_fp64_and_clip_is_the_oracle():
    rs = np.random.RandomState(7)
    v = rs.randn(9, 500)
    for rule in RULES:
        got = AO.resilient_aggregation(v.astype(np.float32), 3, rule)
        assert got.dtype == np.float32
        np.testing.assert_allclose(got, AO.resilient_aggregation(v, 3, rule), rtol=1e-5, atol=1e-6)
    for dt in (np.float32, np.float64):
        np.testing.assert_array_equal(AO.resilient_aggregation(v.astype(dt), 3), O.resilient_aggregation(v.astype(dt), 3))


def test_oracle_refuses_what_the_library_refuses():
    v = np.zeros((4, 2))
    with pytest.raises(ValueError):
        AO.resilient_aggregation(v, 2, "trim")                          # 2H >= n
    with pytest.raises(ValueError):
        AO.resilient_aggregation(v, 4, "wmsr")
    with pytest.raises(ValueError):
        AO.resilient_aggregation(v, 1, "median")


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_rule_field_layout_as_gcc_sees_the_header(tmp_path):
    """`rule` sits in the former tail padding: the job sizes stay 104 / 128 bytes, and the ctypes mirrors agree."""
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'printf("%zu %zu %zu %zu %d %d %d\\n", sizeof(rcmarl_consensus_job), offsetof(rcmarl_consensus_job, rule),'
                   'sizeof(rcmarl_team_job), offsetof(rcmarl_team_job, rule), RCMARL_AGG_CLIP, RCMARL_AGG_TRIM, RCMARL_AGG_WMSR);'
                   'return 0;}')
    exe = tmp_path / "off"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [104, 100, 128, 124, 0, 1, 2]
    assert [ctypes.sizeof(L.ConsensusJob), L.ConsensusJob.rule.offset] == [104, 100]
    assert [ctypes.sizeof(L.TeamJob), L.TeamJob.rule.offset] == [128, 124]
    assert (L.AGG_CLIP, L.AGG_TRIM, L.AGG_WMSR) == (0, 1, 2)
    assert L.ConsensusJob().rule == L.AGG_CLIP and L.TeamJob().rule == L.AGG_CLIP


def test_rule_names_and_limits():
    from rcmarl import _lib as L
    assert [L.agg_rule(r) for r in ("clip", "trim", "wmsr", 1)] == [0, 1, 2, 1]
    with pytest.raises(L.RcmarlError):
        L.agg_rule("median")
    ok = [("clip", 3, 4), ("wmsr", 3, 4), ("trim", 1, 3), ("trim", 7, 15), ("trim", 0, 1), ("wmsr", 0, 16)]
    bad = [("clip", 4, 4), ("wmsr", -1, 4), ("trim", 2, 4), ("trim", 1, 2), ("wmsr", 0, 17), ("clip", 0, 0), (3, 0, 4)]
    for rule, H, n in ok:
        L.check_aggregation(rule, H, n)
    for rule, H, n in bad:
        with pytest.raises(L.RcmarlError):
            L.check_aggregation(rule, H, n)


@pytest.fixture
def no_device(monkeypatch):
    """Trainer construction that reaches the device fails with DeviceTouched instead."""
    import torch
    from rcmarl import _lib

    _lib.lib()                                           # the library is built; Trainer loads it before validating

    class DeviceTouched(Exception):
        pass

    def touched(*a, **k):
        raise DeviceTouched()
    monkeypatch.setattr(torch.cuda, "current_device", touched)
    return DeviceTouched


def trainer(aggregation, H=1, in_nodes=None, labels=None):
    from rcmarl.trainer import Trainer
    labels = labels or ["Cooperative"] * 4 + ["Malicious"]
    in_nodes = in_nodes or [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
    return Trainer(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation)


@pytest.mark.parametrize("aggregation,H", [
    ("median", 1),                                         # unknown name
    (7, 1),                                                # unknown id
    ("trim", 2),                                           # 2H >= n_in = 4
    (["clip", "clip", "trim", "wmsr", "clip"], [1, 1, 2, 1, 0]),   # agent 2: trim with 2H >= 4
    (["clip", "wmsr", "clip", "clip", "clip"], [0, 4, 0, 0, 0]),   # agent 1: H >= n_in
    (["clip", "trim"], 1),                                 # not one rule per agent
])
def test_trainer_refuses_invalid_rules_before_any_device_work(no_device, aggregation, H):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(aggregation, H)


@pytest.mark.parametrize("aggregation,H", [
    ("clip", 1), ("trim", 1), ("wmsr", 3),
    (["trim", "wmsr", "clip", "wmsr", "trim"], [1, 1, 1, 1, 3]),   # the Malicious agent's rule and H are never used
])
def test_trainer_accepts_valid_rules(no_device, aggregation, H):
    with pytest.raises(no_device):
        trainer(aggregation, H)
