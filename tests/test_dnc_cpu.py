"""CPU checks of the divide-and-conquer rule (rcmarl_dnc_aggregate, include/rcmarl.h): properties of the oracle's rule
and weights (tests/dnc_oracle.py), a hand-worked example, the enum and symbol as the header and the bindings declare
them, the library's refusals without a device, and the Trainer's refusals and acceptance before it touches a device.

Selections are compared under a transformation only where they are well defined: a relative eigengap
(lambda_1 - lambda_2) / lambda_1 of at least 1e-3 and a relative score gap at the removal boundary of at least 1e-6."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import assume, given, settings, strategies as st

import dnc_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = (np.inf, -np.inf)
EIG_GAP, SCORE_GAP = 1e-3, 1e-6


@st.composite
def case(draw):
    """(H, X [n, P] float64 from a seeded normal draw around a common centre, each row with its own spread)."""
    H = draw(st.integers(0, 15))
    n = draw(st.integers(H + 1, 16))
    P = draw(st.integers(1, 40))
    rs = np.random.RandomState(draw(st.integers(0, 2 ** 31 - 1)))
    X = rs.randn(n, P) * rs.uniform(0.1, 3, size=(n, 1)) + rs.randn(P) * rs.uniform(0, 100)
    return H, X


def clear(X, H):
    eig, gap = DO.margins(X, H)
    return eig >= EIG_GAP and gap >= SCORE_GAP


@given(case())
@settings(max_examples=300, deadline=None)
def test_weights_are_convex_uniform_on_the_kept_rows_and_give_the_output(c):
    H, X = c
    out, w = DO.aggregate(X, H)
    kept = w > 0
    assert w.shape == (X.shape[0],) and (w >= 0).all() and kept.sum() == X.shape[0] - H
    assert (w[kept] == 1.0 / kept.sum()).all()
    np.testing.assert_allclose(w.sum(), 1.0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(out, w @ X, rtol=1e-9, atol=1e-9 * np.abs(X).max())
    assert sorted(DO.removed(X, H)) == list(np.flatnonzero(~kept))


@given(case())
@settings(max_examples=200, deadline=None)
def test_H0_gives_the_mean(c):
    _, X = c
    out, w = DO.aggregate(X, 0)
    np.testing.assert_allclose(out, X.mean(0), rtol=1e-12, atol=1e-12 * np.abs(X).max())
    np.testing.assert_array_equal(w, np.full(X.shape[0], 1.0 / X.shape[0]))


@given(case(), st.data())
@settings(max_examples=300, deadline=None)
def test_selection_is_unchanged_by_translation_scaling_and_neighbour_permutations(c, data):
    H, X = c
    assume(clear(X, H))
    _, w = DO.aggregate(X, H)
    rs = np.random.RandomState(data.draw(st.integers(0, 1000)))
    t = rs.randn(X.shape[1]) * 50
    a = float(np.exp(rs.uniform(-3, 3)))
    np.testing.assert_array_equal(DO.aggregate(X + t, H)[1], w)
    np.testing.assert_array_equal(DO.aggregate(X * a, H)[1], w)
    p = [0] + list(data.draw(st.permutations(range(1, X.shape[0]))))        # own stays first
    np.testing.assert_array_equal(DO.aggregate(X[p], H)[1], w[p])


@given(st.data())
@settings(max_examples=300, deadline=None)
def test_up_to_H_rows_with_inf_get_weight_zero(data):
    """Up to H rows holding +-inf (whole or in some coordinates) get weight 0 and the output stays finite; if every
    row is flagged, the output is the own row."""
    H = data.draw(st.integers(0, 15))
    n = data.draw(st.integers(H + 1, 16))
    P = data.draw(st.integers(1, 12))
    rs = np.random.RandomState(data.draw(st.integers(0, 2 ** 31 - 1)))
    X = rs.randn(n, P)
    n_bad = data.draw(st.integers(0, H))
    bad = data.draw(st.lists(st.sampled_from(range(n)), min_size=n_bad, max_size=n_bad, unique=True))
    for k in bad:
        cols = data.draw(st.lists(st.sampled_from(range(P)), min_size=1, max_size=P, unique=True))
        for p in cols:
            X[k, p] = data.draw(st.sampled_from(BAD))
    for dt in (np.float64, np.float32):
        out, w = DO.aggregate(X.astype(dt), H)
        assert np.isfinite(out).all(), (H, n, bad)
        assert (w[bad] == 0).all() and w.sum() > 0.99, (H, n, bad, w)
    X[:] = np.inf
    out, w = DO.aggregate(X, H)
    np.testing.assert_array_equal(w, np.eye(n)[0])
    assert np.isinf(out).all()


@given(st.integers(0, 2 ** 31 - 1), st.integers(3, 16), st.data())
@settings(max_examples=200, deadline=None)
def test_a_single_huge_outlier_gets_weight_zero(seed, n, data):
    rs = np.random.RandomState(seed)
    P = rs.randint(1, 40)
    H = data.draw(st.integers(1, n - 1))
    X = rs.randn(n, P)
    k = data.draw(st.integers(0, n - 1))
    X[k, rs.randint(P)] = data.draw(st.sampled_from((1e30, -1e30)))
    for dt in (np.float64, np.float32):
        out, w = DO.aggregate(X.astype(dt), H)
        assert w[k] == 0 and np.isfinite(out).all() and np.abs(out).max() < 10, (n, H, k, w)


def test_fp32_matches_fp64():
    rs = np.random.RandomState(5)
    n_cmp = 0
    for n, H in ((4, 1), (6, 2), (9, 3), (16, 7)):
        X = rs.randn(n, 700) * rs.uniform(0.2, 2, size=(n, 1)) + rs.randn(700)
        if not clear(X, H):
            continue
        o32, w32 = DO.aggregate(X.astype(np.float32), H)
        o64, w64 = DO.aggregate(X, H)
        assert o32.dtype == np.float32
        np.testing.assert_array_equal(w32 > 0, w64 > 0)
        np.testing.assert_allclose(o32, o64, rtol=1e-5, atol=1e-5)
        n_cmp += 1
    assert n_cmp >= 3


def test_hand_worked_example():
    """Five collinear messages x_k = t_k e + b: the centred rows are (t_k - 2) e, so G has rank one, lambda = 106 and
    score_k = (t_k - 2)^2 = 4, 1, 1, 36, 64.  H = 1 removes row 4, H = 2 also row 3, H = 3 also the own row 0."""
    t = np.array([0.0, 1.0, 3.0, -4.0, 10.0])
    e, b = np.array([0.6, 0.8]), np.array([5.0, -2.0])
    X = t[:, None] * e + b
    np.testing.assert_allclose(DO.scores(X), [4, 1, 1, 36, 64], rtol=1e-12)
    lam, _ = DO.spectrum(X)
    np.testing.assert_allclose(lam[-1], 106, rtol=1e-12)
    for H, keep in ((0, [0, 1, 2, 3, 4]), (1, [0, 1, 2, 3]), (2, [0, 1, 2]), (3, [1, 2])):
        out, w = DO.aggregate(X, H)
        want = np.zeros(5)
        want[keep] = 1.0 / len(keep)
        np.testing.assert_array_equal(w, want)
        np.testing.assert_allclose(out, X[keep].mean(0), rtol=1e-14)


def test_oracle_refuses_what_the_library_refuses():
    X = np.zeros((4, 3))
    for H in (-1, 4, 5):
        with pytest.raises(ValueError):
            DO.aggregate(X, H)


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enum_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "dnc.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_vector_job*, int, void*) = rcmarl_dnc_aggregate; (void)f;'
                   'printf("%d %d %d\\n", RCMARL_SPECTRAL_DNC, RCMARL_DNC_SWEEPS, RCMARL_DNC_MAX_FLOATS); return 0;}')
    exe = tmp_path / "dnc"
    # links against nothing: only the declaration's type is checked, so compile to an object and print from a stub
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_dnc_aggregate(const rcmarl_vector_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [L.SPECTRAL_DNC, L.DNC_SWEEPS, L.DNC_MAX_FLOATS] == [0, 32, 48 * 1024]
    assert L.SPECTRAL_RULES == {"dnc": 0}
    assert ("rcmarl_dnc_aggregate", ctypes.c_int, [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_dnc_aggregate.argtypes == [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 rows of 100 floats, 1000 floats apart, dst far away."""
    from rcmarl import _lib as L
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = 1 << 24, 1 << 16, 1000, 100, 4, 1, L.SPECTRAL_DNC
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
    dict(rule=1), dict(rule=-1), dict(rule=4), dict(H=-1), dict(H=4), dict(n_in=1, H=1),
    dict(n=48 * 1024 // 6 + 1),                                              # (n_in + 2) * n over the staging limit
    dict(dst=(1 << 16) + 4 * 2000), dict(dst=(1 << 16) + 4 * 2000 + 396), dict(dst=(1 << 16) - 4 * 99),   # overlaps rows
    dict(weights_out=(1 << 16) + 4 * 1000 + 8), dict(weights_out=(1 << 16) - 4 * 3),   # weights_out on an in-node row
    dict(weights_out=(1 << 24) + 4 * 99),                                            # ... or on the job's own dst
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    for jobs in ([_job(**bad)], [_job(dst=1 << 26, weights_out=(1 << 26) + 4096), _job(**bad)]):
        arr = (L.VectorJob * len(jobs))(*jobs)
        assert lib.rcmarl_dnc_aggregate(arr, len(arr), None) == -1                   # RCMARL_ERR_ARG


def test_library_refuses_writes_on_another_jobs_ranges_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    arr = (L.VectorJob * 2)(_job(msgs=1 << 28), _job(dst=(1 << 28) + 4 * 1000))   # job 1 writes job 0's row 1
    assert lib.rcmarl_dnc_aggregate(arr, 2, None) == -1
    first = dict(dst=1 << 26, weights_out=(1 << 26) + 4096)
    for second in (dict(dst=(1 << 26) + 4 * 99), dict(weights_out=(1 << 26) + 4 * 50), dict(weights_out=(1 << 26) + 4096 + 12),
                   dict(dst=(1 << 26) + 4096 - 8)):
        arr = (L.VectorJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_dnc_aggregate(arr, 2, None) == -1, second
    assert lib.rcmarl_dnc_aggregate(None, 1, None) == -1
    arr = (L.VectorJob * 33)(*[_job(dst=(1 << 24) + 4096 * i) for i in range(33)])
    assert lib.rcmarl_dnc_aggregate(arr, 0, None) == -1
    assert lib.rcmarl_dnc_aggregate(arr, 33, None) == -1


def test_rule_names_and_limits():
    from rcmarl import _lib as L
    for H, n in ((0, 1), (1, 2), (15, 16), (0, 16)):
        assert L.check_spectral_rule(H, n) == 0
    for H, n in ((1, 1), (-1, 4), (4, 4), (0, 0), (0, 17)):
        with pytest.raises(L.RcmarlError):
            L.check_spectral_rule(H, n)
    assert L.is_spectral_rule("dnc") and not L.is_spectral_rule("DnC") and not L.is_spectral_rule(0)
    assert not L.is_vector_rule("dnc") and "dnc" not in L.AGG_RULES


# ------------------------------------------------------------------------------------------------ Trainer
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
BYZ = ["Cooperative"] * 4 + ["Byzantine"]


def trainer(aggregation, H=1, labels=None, attack=None):
    from rcmarl.trainer import Trainer
    labels = labels or ["Cooperative"] * 4 + ["Malicious"]
    return Trainer(labels=labels, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack)


@pytest.mark.parametrize("aggregation,H,labels,attack", [
    ("dnc", 4, None, None),                                                   # H >= n_in
    ("dnc", [0, 5, 0, 0, 0], None, None),
    (["dnc", "clip", "dnc", "clip", "clip"], [1, 0, -1, 0, 0], None, None),
    ("DnC", 1, None, None),
    ("dnc", 1, BYZ, ("tailored_std", 2.0)),                                  # the tailored attack does not model dnc
    (["clip", "clip", "dnc", "clip", "clip"], 1, BYZ, ("tailored_uv", 2.0)),  # ... at one receiver of agent 4
])
def test_trainer_refuses_before_any_device_work(no_device, aggregation, H, labels, attack):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(aggregation, H, labels, attack)


@pytest.mark.parametrize("aggregation,H,labels,attack", [
    ("dnc", 0, None, None), ("dnc", 3, None, None),
    (["dnc", "trim", "krum", "wmsr", "clip"], [1, 1, 1, 1, 0], None, None),
    (["gmed", "dnc", "clip", "mkrum", "scclip"], [1, 2, 1, 1, 9], BYZ, ("minmax_uv", 1.0)),
    (["dnc", "dnc", "scclip", "trim", "clip"], [3, 2, 1, 1, 0], BYZ, ("alie", 1.0)),
    (["dnc", "clip", "clip", "clip", "clip"], 1, BYZ, ("tailored_std", 2.0)),   # agent 0 does not hear agent 4
])
def test_trainer_accepts_dnc_alone_and_mixed(no_device, aggregation, H, labels, attack):
    with pytest.raises(no_device):
        trainer(aggregation, H, labels, attack)
