"""The iterative outlier scissor (rcmarl_ios_aggregate, include/rcmarl.h) without a GPU: the NumPy oracle
(tests/ios_oracle.py) on a hand-worked example and its invariances, the C ABI as gcc sees it, the library's refusals on
made-up addresses, the binding's names and limits, and the Trainer's checks before any device work."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import ios_oracle as IO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ oracle
def test_recentring_removes_a_different_row_than_one_shot_removal():
    """Honest rows 0, 0, 0, -4 and outliers 6 and 30 at H = 2.  The first mean, 16/3, is pulled towards 30, so 6 lies
    next to it and the honest -4 far off: removing the two rows furthest from that one mean drops 30 and -4.  IOS drops
    30, re-centres at 0.4 and then drops 6 (d = 31.36 against 19.36 for -4)."""
    X = np.array([[0.0], [0.0], [0.0], [-4.0], [6.0], [30.0]])
    d0 = IO.distances(X, range(6))
    one_shot = sorted(sorted(range(6), key=lambda k: -d0[k])[:2])
    assert one_shot == [3, 5]
    st = IO.steps(X, 2)
    assert [top for _, _, top in st] == [5, 4]
    assert st[1][1][4] == pytest.approx(31.36) and st[1][1][3] == pytest.approx(19.36)
    out, w = IO.aggregate(X, 2)
    assert IO.kept(X, 2) == (0, 1, 2, 3)
    np.testing.assert_array_equal(w, [0.25, 0.25, 0.25, 0.25, 0, 0])
    np.testing.assert_array_equal(out, [-1.0])
    assert IO.margin(X, 2) > 0.3


@pytest.mark.parametrize("seed", range(8))
def test_weights_are_convex_uniform_on_the_kept_rows_and_give_the_output(seed):
    rs = np.random.RandomState(200 + seed)
    n = int(rs.randint(1, 17))
    H = int(rs.randint(0, n))
    X = (rs.randn(n, 37) * rs.uniform(0.1, 3, size=(n, 1))).astype(np.float32)
    out, w = IO.aggregate(X, H)
    keep = w > 0
    assert keep.sum() == n - H and (w[keep] == np.float32(1) / np.float32(n - H)).all() and (w[~keep] == 0).all()
    assert abs(float(w.astype(np.float64).sum()) - 1.0) < 1e-6
    np.testing.assert_array_equal(out, IO.mean_of(X, np.flatnonzero(keep)))
    np.testing.assert_allclose(out, (w.astype(np.float64) @ X.astype(np.float64)), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_H0_gives_the_plain_mean(dt):
    rs = np.random.RandomState(3)
    for n in (1, 2, 5, 16):
        X = rs.randn(n, 33).astype(dt)
        out, w = IO.aggregate(X, 0)
        want = np.zeros(33, dt)
        for k in range(n):
            want = want + X[k]
        np.testing.assert_array_equal(out, want / dt(n))
        np.testing.assert_array_equal(w, np.full(n, dt(1) / dt(n)))
        assert IO.steps(X, 0) == []


@pytest.mark.parametrize("seed", range(6))
def test_selection_is_invariant_under_translation_scaling_and_permutation(seed):
    """Away from ties (margin above 1e-6), the kept set moves with the rows: x -> a x + b (a > 0) keeps the same rows,
    and permuting the neighbours permutes the kept set.  H <= n - 2: two rows left tie in exact arithmetic, and the
    affine map rounds their fp64 sums."""
    rs = np.random.RandomState(300 + seed)
    n = int(rs.randint(3, 17))
    H = int(rs.randint(1, n - 1))
    X = rs.randn(n, 25) * rs.uniform(0.2, 3, size=(n, 1))
    assert IO.margin(X, H) > 1e-6
    sel = IO.kept(X, H)
    a, b = rs.uniform(0.01, 100), rs.randn(25) * 10
    assert IO.kept(a * X + b, H) == sel
    perm = rs.permutation(n)
    Y = X[perm]                                          # row q of Y is row perm[q] of X
    assert sorted(perm[list(IO.kept(Y, H))]) == list(sel)


def test_equal_distances_remove_the_higher_index_first():
    X = np.array([[1.0, 0.0], [-1.0, 0.0], [0.0, 1.0], [0.0, -1.0]])   # every row at distance 1 from the centre 0
    assert [top for _, _, top in IO.steps(X, 1)] == [3]
    assert IO.kept(X, 1) == (0, 1, 2)
    X = np.tile(np.array([[1.5, -2.0, 3.0]]), (6, 1))
    for H in range(6):
        assert IO.kept(X, H) == tuple(range(6 - H))
        assert IO.margin(X, H) == np.inf                 # equal rows tie in any precision


@pytest.mark.parametrize("seed", range(8))
def test_up_to_H_bad_rows_get_weight_zero(seed):
    rs = np.random.RandomState(100 + seed)
    n = int(rs.randint(3, 17))
    H = int(rs.randint(1, (n - 1) // 2 + 1))
    X = rs.randn(n, 20) * rs.uniform(0.1, 1, size=(n, 1))
    nb = int(rs.randint(1, H + 1))
    bad = rs.choice(n, size=nb, replace=False)
    for k in bad:
        cols = rs.choice(20, size=int(rs.randint(1, 21)), replace=False)
        X[k, cols] = rs.choice([1e30, -1e30, np.inf, -np.inf])
    out, w = IO.aggregate(X, H)
    assert (w[bad] == 0).all() and np.isfinite(out).all()
    assert (w > 0).sum() == n - max(H, int(IO.flagged(X).sum()))


def test_every_row_flagged_gives_the_own_row():
    X = np.array([[np.inf, 1.0], [2.0, -np.inf], [np.inf, np.inf]])
    out, w = IO.aggregate(X, 1)
    np.testing.assert_array_equal(out, X[0])
    np.testing.assert_array_equal(w, [1, 0, 0])


def test_more_flagged_rows_than_H_remove_every_flagged_row_and_nothing_else():
    X = np.array([[0.0, 0.0], [np.inf, 0.0], [1.0, 1.0], [-np.inf, 2.0], [50.0, 50.0]])
    assert IO.steps(X, 1) == [] and IO.kept(X, 1) == (0, 2, 4)
    assert [top for _, _, top in IO.steps(X, 3)] == [4] and IO.kept(X, 3) == (0, 2)


def test_oracle_refuses_what_the_library_refuses():
    X = np.zeros((4, 3))
    for H in (-1, 4, 5):
        with pytest.raises(ValueError):
            IO.aggregate(X, H)


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enum_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "ios.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_vector_job*, int, void*) = rcmarl_ios_aggregate; (void)f;'
                   'rcmarl_filter_rule r = RCMARL_FILTER_IOS;'
                   'printf("%d %d\\n", (int)r, RCMARL_IOS_MAX_FLOATS); return 0;}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_ios_aggregate(const rcmarl_vector_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "ios"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [L.FILTER_IOS, L.IOS_MAX_FLOATS] == [0, 48 * 1024]
    assert (16 + 2) * 1421 <= L.IOS_MAX_FLOATS               # the 16-agent team-reward net at n_in = 16
    assert ("rcmarl_ios_aggregate", ctypes.c_int, [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_ios_aggregate.argtypes == [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 rows of 100 floats, 1000 floats apart, dst far away."""
    from rcmarl import _lib as L
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = 1 << 24, 1 << 16, 1000, 100, 4, 1, L.FILTER_IOS
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
    dict(rule=1), dict(rule=-1), dict(H=-1), dict(H=4), dict(n_in=1, H=1),
    dict(n=48 * 1024 // 6 + 1),                                              # (n_in + 2) * n over the staging bound
    dict(n_in=1, H=0, n=48 * 1024 // 3 + 1),                                 # ... by one float's worth of rows
    dict(dst=(1 << 16) + 4 * 2000), dict(dst=(1 << 16) + 4 * 2000 + 396), dict(dst=(1 << 16) - 4 * 99),   # overlaps rows
    dict(weights_out=(1 << 16) + 4 * 1000 + 8), dict(weights_out=(1 << 16) - 4 * 3),   # weights_out on an in-node row
    dict(weights_out=(1 << 24) + 4 * 99),                                            # ... or on the job's own dst
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    bad_job = _job(**bad)
    for jobs in ([bad_job], [_job(dst=1 << 26, weights_out=(1 << 26) + 4096), bad_job]):
        arr = (L.VectorJob * len(jobs))(*jobs)
        assert lib.rcmarl_ios_aggregate(arr, len(arr), None) == -1               # RCMARL_ERR_ARG


def test_library_refuses_writes_on_another_jobs_ranges_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    arr = (L.VectorJob * 2)(_job(msgs=1 << 28), _job(dst=(1 << 28) + 4 * 1000))   # job 1 writes job 0's row 1
    assert lib.rcmarl_ios_aggregate(arr, 2, None) == -1
    first = dict(dst=1 << 26, weights_out=(1 << 26) + 4096)
    for second in (dict(dst=(1 << 26) + 4 * 99), dict(weights_out=(1 << 26) + 4 * 50),
                   dict(weights_out=(1 << 26) + 4096 + 12), dict(dst=(1 << 26) + 4096 - 8)):
        arr = (L.VectorJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_ios_aggregate(arr, 2, None) == -1, second
    assert lib.rcmarl_ios_aggregate(None, 1, None) == -1
    arr = (L.VectorJob * 33)(*[_job(dst=(1 << 24) + 4096 * i) for i in range(33)])
    assert lib.rcmarl_ios_aggregate(arr, 0, None) == -1
    assert lib.rcmarl_ios_aggregate(arr, 33, None) == -1


def test_rule_names_and_limits():
    from rcmarl import _lib as L
    assert L.FILTER_RULES == {"ios": 0} and L.FILTER_IOS == 0
    for H, n in ((0, 1), (1, 2), (15, 16), (0, 16), (7, 16)):
        assert L.check_filter_rule(H, n) == L.FILTER_IOS
    for H, n in ((1, 1), (-1, 4), (4, 4), (0, 0), (0, 17)):
        with pytest.raises(L.RcmarlError):
            L.check_filter_rule(H, n)
    assert L.is_filter_rule("ios")
    assert not L.is_filter_rule("IOS") and not L.is_filter_rule(0) and not L.is_filter_rule("dnc")
    assert not L.is_vector_rule("ios") and not L.is_spectral_rule("ios") and not L.is_subset_rule("ios")
    assert "ios" not in L.AGG_RULES


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


def trainer(aggregation, H=1, labels=None, attack=None, mixing=None, momentum=None, clipping=None):
    from rcmarl.trainer import Trainer
    labels = labels or ["Cooperative"] * 4 + ["Malicious"]
    return Trainer(labels=labels, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing, momentum=momentum, clipping=clipping)


@pytest.mark.parametrize("aggregation,H,mixing", [
    ("ios", 4, None),                                                        # H >= n_in
    ("ios", [0, 5, 0, 0, 0], None),
    (["ios", "clip", "ios", "clip", "clip"], [1, 0, -1, 0, 0], None),
    ("IOS", 1, None),
    ("ios", 3, ("bucket", 2)),                                               # 3 bucket rows leave H = 3 >= n_out
    (["clip", "ios", "clip", "clip", "clip"], 2, ("bucket", 3)),             # 2 rows
])
def test_trainer_refuses_bad_rules_before_any_device_work(no_device, aggregation, H, mixing):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(aggregation, H, mixing=mixing)


@pytest.mark.parametrize("attack", ["tailored_std", "pipeline_uv", "history_std", "arc_sgn", "subset_std"])
@pytest.mark.parametrize("receiver", [1, 3])
def test_trainer_refuses_rule_aware_attacks_against_an_ios_receiver_before_any_device_work(no_device, attack,
                                                                                           receiver):
    """Agents 1, 2 and 3 hear Byzantine agent 4; the one on ios refuses every rule-aware family, by name."""
    from rcmarl import _lib as L
    agg = ["clip"] * 5
    agg[receiver] = "ios"
    with pytest.raises(L.RcmarlError, match=rf"Byzantine agent 4 runs .* against agent {receiver}, whose rule 'ios'"):
        trainer(agg, 1, BYZ, (attack, 2.0))


@pytest.mark.parametrize("aggregation,H,labels,attack,mixing,momentum,clipping", [
    ("ios", 0, None, None, None, None, None), ("ios", 3, None, None, None, None, None),
    (["ios", "trim", "krum", "ios", "clip"], [1, 1, 1, 1, 0], None, None, None, None, None),
    (["gmed", "ios", "dnc", "mkrum", "mda"], [1, 2, 1, 1, 9], BYZ, ("minmax_std", 1.0), None, None, None),
    (["ios", "smea", "scclip", "wmsr", "clip"], [3, 2, 1, 1, 0], BYZ, ("alie", 1.0), "nnm", None, None),
    (["ios", "ios", "dnc", "clip", "clip"], 1, BYZ, ("ipm", 0.5), ("bucket", 2), None, None),
    ("ios", 1, BYZ, ("gauss", 0.3), None, 0.9, None),
    ("ios", 1, BYZ, ("dissensus", 1.0), None, None, "arc"),
    (["ios", "ios", "clip", "clip", "clip"], 1, BYZ, ("mimic", 2), [("bucket", 2), "nnm", None, None, None], None,
     "arc"),
    ("ios", 2, BYZ, ("minsum_uv", 1.0), None, [0.5, 0.9, None, 0.99, None], ["arc", None, "arc", "arc", None]),
    (["ios", "clip", "clip", "clip", "clip"], 1, BYZ, ("tailored_std", 2.0), None, None, None),   # 0 does not hear 4
    (["ios", "clip", "clip", "clip", "clip"], 1, BYZ, ("subset_uv", 2.0), None, None, "arc"),    # ... nor here
])
def test_trainer_accepts_ios_alone_mixed_and_composed(no_device, aggregation, H, labels, attack, mixing, momentum,
                                                      clipping):
    with pytest.raises(no_device):
        trainer(aggregation, H, labels, attack, mixing, momentum, clipping)
