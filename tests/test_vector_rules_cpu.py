"""CPU checks of the distance-based resilient aggregation rules (rcmarl_vector_rule: krum, mkrum, scclip, gmed,
include/rcmarl.h): properties of the oracle's rules and weights (tests/vector_oracle.py), the C layout of the job and the
ctypes mirror, the library's refusals without a device, and the Trainer's refusal of an invalid rule before it touches
a device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import HealthCheck, assume, given, settings, strategies as st

import vector_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULES = VO.RULES
BAD = (1e30, -1e30, np.inf, -np.inf)


def min_n(rule, H):
    return H + 3 if rule in ("krum", "mkrum") else H + 1


@st.composite
def case(draw, rules=RULES):
    """(rule, H, X [n, P] float64 from a seeded normal draw: continuous, so no two scores tie)."""
    rule = draw(st.sampled_from(rules))
    H = draw(st.integers(0, 6))
    n = draw(st.integers(min_n(rule, H), 16))
    P = draw(st.integers(1, 40))
    rs = np.random.RandomState(draw(st.integers(0, 2 ** 31 - 1)))
    X = rs.randn(n, P) * rs.uniform(0.1, 10) + rs.randn(P) * rs.uniform(0, 100)
    return rule, H, X


@given(case())
@settings(max_examples=300, deadline=None)
def test_weights_are_convex_and_give_the_output(c):
    rule, H, X = c
    out, w = VO.aggregate(X, H, rule)
    assert w.shape == (X.shape[0],) and (w >= 0).all()
    np.testing.assert_allclose(w.sum(), 1.0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(out, w @ X, rtol=1e-9, atol=1e-9 * np.abs(X).max())


@given(case(rules=("scclip", "mkrum")))
@settings(max_examples=200, deadline=None)
def test_H0_scclip_and_mkrum_give_the_mean(c):
    rule, _, X = c
    out, w = VO.aggregate(X, 0, rule)
    np.testing.assert_allclose(out, X.mean(0), rtol=1e-12, atol=1e-12 * np.abs(X).max())
    np.testing.assert_allclose(w, np.full(X.shape[0], 1.0 / X.shape[0]), rtol=0, atol=1e-14)


@given(case(), st.data())
@settings(max_examples=200, deadline=None, suppress_health_check=[HealthCheck.filter_too_much])
def test_equivariant_under_translation_and_neighbour_permutations(c, data):
    rule, H, X = c
    out, w = VO.aggregate(X, H, rule)
    scale = np.abs(X).max()
    t = np.random.RandomState(data.draw(st.integers(0, 1000))).randn(X.shape[1]) * 50
    out_t, w_t = VO.aggregate(X + t, H, rule)
    np.testing.assert_allclose(out_t, out + t, rtol=1e-7, atol=1e-7 * (scale + 50 * 5))
    np.testing.assert_allclose(w_t, w, rtol=1e-6, atol=1e-9)
    if rule in ("krum", "mkrum"):
        # mutual nearest neighbours have equal scores (D is symmetric), and a tie at the selection boundary goes to the
        # lower index, which a permutation changes
        m = 1 if rule == "krum" else X.shape[0] - H
        s = np.sort(VO.krum_scores(X, H))
        assume(m == X.shape[0] or s[m] - s[m - 1] > 1e-9 * s[m])
    p = [0] + list(data.draw(st.permutations(range(1, X.shape[0]))))        # own stays first
    out_p, w_p = VO.aggregate(X[p], H, rule)
    np.testing.assert_allclose(out_p, out, rtol=1e-9, atol=1e-9 * scale)
    np.testing.assert_allclose(w_p, w[p], rtol=1e-9, atol=1e-12)


@given(st.sampled_from(RULES), st.data())
@settings(max_examples=300, deadline=None)
def test_at_most_H_byzantine_messages_get_weight_zero(rule, data):
    """Up to H messages of 1e30 / +-inf (whole or in some coordinates) get weight 0 and the output stays finite, while
    the rule's guarantee holds: n >= 2H + 3 for krum / mkrum, 2H < n for gmed, H < n for scclip."""
    H = data.draw(st.integers(0, {"krum": 6, "mkrum": 6, "gmed": 7, "scclip": 15}[rule]))
    n = data.draw(st.integers({"krum": 2 * H + 3, "mkrum": 2 * H + 3, "gmed": 2 * H + 1, "scclip": H + 1}[rule], 16))
    P = data.draw(st.integers(1, 12))
    rs = np.random.RandomState(data.draw(st.integers(0, 2 ** 31 - 1)))
    X = rs.randn(n, P)
    n_bad = data.draw(st.integers(0, min(H, n - 1)))
    bad = data.draw(st.lists(st.sampled_from(range(1, n)), min_size=n_bad, max_size=n_bad, unique=True)) if n > 1 else []
    for k in bad:
        cols = data.draw(st.lists(st.sampled_from(range(P)), min_size=1, max_size=P, unique=True))
        for p in cols:
            X[k, p] = data.draw(st.sampled_from(BAD))
    for dt in (np.float64, np.float32):
        out, w = VO.aggregate(X.astype(dt), H, rule)
        assert np.isfinite(out).all(), (rule, H, n, bad)
        assert (w[bad] == 0).all(), (rule, H, n, bad, w)
        honest = np.delete(X, bad, axis=0)
        assert (out >= honest.min(0) - 1e-3).all() and (out <= honest.max(0) + 1e-3).all()


@given(st.integers(0, 2 ** 31 - 1), st.integers(1, 7))
@settings(max_examples=200, deadline=None)
def test_gmed_of_collinear_points_is_their_median(seed, half):
    rs = np.random.RandomState(seed)
    n = 2 * half + 1                                                  # odd: the median point is unique
    P = rs.randint(1, 30)
    t = rs.randn(n) * 3
    t[rs.randint(n)] += 0.5                                           # distinct positions
    u, c = rs.randn(P), rs.randn(P) * 10
    X = t[:, None] * u + c
    out, _ = VO.aggregate(X, 0, "gmed")
    np.testing.assert_allclose(out, np.median(t) * u + c, rtol=0, atol=1e-4 * (1 + np.abs(X).max()))


def test_krum_picks_the_centre_of_a_cluster_and_mkrum_averages_it():
    X = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 1.1], [50.0, 50.0], [-0.2, 0.1]])
    out, w = VO.aggregate(X, 1, "krum")
    # scores (the n - H - 2 = 2 smallest squared distances): 1.05, 2.45, 2.25, 4891.21 + 4901, 1.09
    np.testing.assert_allclose(VO.krum_scores(X, 1), [1.05, 2.45, 2.25, 9792.21, 1.09])
    np.testing.assert_array_equal(w, [1, 0, 0, 0, 0])
    np.testing.assert_array_equal(out, X[0])
    out, w = VO.aggregate(X, 1, "mkrum")
    np.testing.assert_array_equal(w > 0, [True, True, True, False, True])
    np.testing.assert_allclose(out, X[[0, 1, 2, 4]].mean(0))


def test_fp32_matches_fp64():
    rs = np.random.RandomState(3)
    X = rs.randn(9, 700)
    for rule in RULES:
        o32, w32 = VO.aggregate(X.astype(np.float32), 2, rule)
        o64, w64 = VO.aggregate(X, 2, rule)
        assert o32.dtype == np.float32
        np.testing.assert_allclose(o32, o64, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(w32, w64, rtol=1e-4, atol=1e-6)


def test_oracle_refuses_what_the_library_refuses():
    X = np.zeros((4, 3))
    for rule, H in (("krum", 2), ("mkrum", 2), ("scclip", 4), ("gmed", -1), ("median", 0)):
        with pytest.raises(ValueError):
            VO.aggregate(X, H, rule)


# ------------------------------------------------------------------------------------------------ C ABI / bindings
FIELDS = ["dst", "msgs", "msg_stride", "weights_out", "n", "n_in", "H", "rule", "in_nodes"]


def test_vector_job_layout_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'printf("%zu", sizeof(rcmarl_vector_job));'
                   + "".join(f'printf(" %zu", offsetof(rcmarl_vector_job, {f}));' for f in FIELDS)
                   + 'printf(" %d %d %d %d %d %d %.17g\\n", RCMARL_VEC_KRUM, RCMARL_VEC_MKRUM, RCMARL_VEC_SCCLIP, '
                   'RCMARL_VEC_GMED, RCMARL_GMED_ITERS, RCMARL_VECTOR_MAX_FLOATS, (double)RCMARL_GMED_NU); return 0;}')
    exe = tmp_path / "off"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = subprocess.check_output([str(exe)]).split()
    sizes = [int(x) for x in got[:1 + len(FIELDS)]]
    assert sizes[0] == ctypes.sizeof(L.VectorJob) == 112
    assert sizes[1:] == [getattr(L.VectorJob, f).offset for f in FIELDS]
    enums = [int(x) for x in got[1 + len(FIELDS):-1]]
    assert enums == [L.VEC_KRUM, L.VEC_MKRUM, L.VEC_SCCLIP, L.VEC_GMED, L.GMED_ITERS, L.VECTOR_MAX_FLOATS]
    assert enums[:5] == [0, 1, 2, 3, VO.GMED_ITERS]
    assert float(got[-1]) == float(np.float32(L.GMED_NU)) and L.GMED_NU == VO.GMED_NU
    assert sorted(L.VECTOR_RULES) == sorted(VO.RULES) and [L.VECTOR_RULES[r] for r in VO.RULES] == [0, 1, 2, 3]
    assert ("rcmarl_vector_aggregate", ctypes.c_int, [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS


def _job(**kw):
    """A valid job on made-up addresses: 4 rows of 100 floats, 1000 floats apart, dst far away."""
    from rcmarl import _lib as L
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = 1 << 24, 1 << 16, 1000, 100, 4, 1, L.VEC_KRUM
    for k in range(4):
        j.in_nodes[k] = k
    for k, v in kw.items():
        if k == "in_nodes":
            for i, x in enumerate(v):
                j.in_nodes[i] = x
        else:
            setattr(j, k, v)
    return j


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-5), dict(n_in=0), dict(n_in=17), dict(in_nodes=[0, 1, -1, 3]),
    dict(rule=4), dict(rule=-1), dict(H=-1), dict(H=4, rule=2), dict(H=2), dict(n_in=2, H=0), dict(rule=1, H=2),
    dict(n=48 * 1024 // 5 + 1),                                              # (n_in + 1) * n over the staging limit
    dict(dst=(1 << 16) + 4 * 2000), dict(dst=(1 << 16) + 4 * 2000 + 396), dict(dst=(1 << 16) - 4 * 99),   # overlaps rows
    dict(weights_out=(1 << 16) + 4 * 1000 + 8), dict(weights_out=(1 << 16) - 4 * 3),   # weights_out on an in-node row
    dict(weights_out=(1 << 24) + 4 * 99),                                            # ... or on the job's own dst
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    for jobs in ([_job(**bad)], [_job(dst=1 << 26, weights_out=(1 << 26) + 4096), _job(**bad)]):
        arr = (L.VectorJob * len(jobs))(*jobs)
        assert lib.rcmarl_vector_aggregate(arr, len(arr), None) == -1                # RCMARL_ERR_ARG


def test_library_refuses_writes_on_another_jobs_ranges_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    arr = (L.VectorJob * 2)(_job(msgs=1 << 28), _job(dst=(1 << 28) + 4 * 1000))   # job 1 writes job 0's row 1
    assert lib.rcmarl_vector_aggregate(arr, 2, None) == -1
    # two jobs whose written ranges (dst, weights_out) overlap: the CTAs of a launch run concurrently
    first = dict(dst=1 << 26, weights_out=(1 << 26) + 4096)
    for second in (dict(dst=(1 << 26) + 4 * 99), dict(weights_out=(1 << 26) + 4 * 50), dict(weights_out=(1 << 26) + 4096 + 12),
                   dict(dst=(1 << 26) + 4096 - 8)):
        arr = (L.VectorJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_vector_aggregate(arr, 2, None) == -1, second
    assert lib.rcmarl_vector_aggregate(None, 1, None) == -1
    arr = (L.VectorJob * 33)(*[_job(dst=(1 << 24) + 4096 * i) for i in range(33)])
    assert lib.rcmarl_vector_aggregate(arr, 0, None) == -1
    assert lib.rcmarl_vector_aggregate(arr, 33, None) == -1


def test_rule_names_and_limits():
    from rcmarl import _lib as L
    assert [L.check_vector_rule(r, 0, 3) for r in ("krum", "mkrum", "scclip", "gmed")] == [0, 1, 2, 3]
    ok = [("krum", 1, 4), ("mkrum", 13, 16), ("scclip", 0, 1), ("scclip", 15, 16), ("gmed", 0, 1), ("gmed", 7, 8)]
    bad = [("krum", 2, 4), ("mkrum", 0, 2), ("scclip", 1, 1), ("gmed", 0, 17), ("gmed", -1, 4), ("median", 0, 4),
           ("clip", 0, 4), (0, 0, 4)]
    for rule, H, n in ok:
        L.check_vector_rule(rule, H, n)
    for rule, H, n in bad:
        with pytest.raises(L.RcmarlError):
            L.check_vector_rule(rule, H, n)
    assert not L.is_vector_rule(0) and not L.is_vector_rule("median") and L.AGG_RULES == {"clip": 0, "trim": 1, "wmsr": 2}


# ------------------------------------------------------------------------------------------------ Trainer refusals
@pytest.fixture
def no_device(monkeypatch):
    """Trainer construction that reaches the device fails with DeviceTouched instead."""
    import torch
    from rcmarl import _lib

    _lib.lib()

    class DeviceTouched(Exception):
        pass

    def touched(*a, **k):
        raise DeviceTouched()
    monkeypatch.setattr(torch.cuda, "current_device", touched)
    return DeviceTouched


C5 = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]


def trainer(aggregation, H=1, labels=None, attack=None):
    from rcmarl.trainer import Trainer
    labels = labels or ["Cooperative"] * 4 + ["Malicious"]
    return Trainer(labels=labels, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack)


@pytest.mark.parametrize("aggregation,H", [
    ("krum", 2),                                                     # n_in = 4 < H + 3
    ("mkrum", [0, 2, 0, 0, 0]),
    (["gmed", "scclip", "krum", "clip", "clip"], [3, 3, 3, 0, 0]),   # agent 2: krum with H = 3
    ("scclip", 4),                                                   # H >= n_in
    ("median", 1),                                                   # unknown names
    ("Krum", 1),
    (["krum", "gmed"], 1),                                           # not one rule per agent
    (["krum"] * 6, 1),
])
def test_trainer_refuses_invalid_vector_rules_before_any_device_work(no_device, aggregation, H):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(aggregation, H)


@pytest.mark.parametrize("aggregation,H,labels,attack", [
    ("krum", 1, None, None), ("mkrum", 1, None, None), ("scclip", 3, None, None), ("gmed", 3, None, None),
    (["krum", "trim", "gmed", "wmsr", "clip"], [1, 1, 3, 2, 0], None, None),    # mixed per agent
    (["scclip", "mkrum", "clip", "gmed", "krum"], [2, 1, 1, 0, 9], ["Cooperative"] * 4 + ["Byzantine"], ("alie", 1.0)),
])
def test_trainer_accepts_valid_and_mixed_rules(no_device, aggregation, H, labels, attack):
    with pytest.raises(no_device):
        trainer(aggregation, H, labels, attack)
