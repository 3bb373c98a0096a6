"""The exact subset-selection rules MDA and SMEA (rcmarl_subset_aggregate, include/rcmarl.h) without a GPU: the NumPy
oracle (tests/subset_oracle.py) on known answers and against brute force, the C ABI as gcc sees it, the library's
refusals on made-up addresses, the binding's names and limits, and the Trainer's checks before any device work."""
import ctypes
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

import subset_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULES = SO.RULES


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("rule", RULES)
def test_collinear_outlier_is_dropped(rule):
    X = np.array([[0.0], [1.0], [2.0], [10.0]])
    out, w = SO.aggregate(rule, X, 1)
    np.testing.assert_array_equal(w, [1 / 3, 1 / 3, 1 / 3, 0])
    np.testing.assert_array_equal(out, [1.0])
    # MDA: diameters 4 (drop 10), 81, 100, 100; SMEA: 2 * the variance along the line
    D = SO.distances(X)
    assert [SO.criterion("mda", D, S) for S in itertools.combinations(range(4), 3)] == [4, 100, 100, 81]


def test_mda_and_smea_disagree_on_a_cluster_with_an_outlier_along_its_spread():
    """Rows 1 and 3 are a tight pair; row 0 lies far off on one side and row 2 on another.  MDA keeps the subset of
    smallest diameter {0, 1, 3} (26 against 29); SMEA the one whose spread is most even, {1, 2, 3}."""
    X = np.array([[0.0, 4.0], [-1.0, -1.0], [-4.0, -3.0], [1.0, -1.0]])
    D = SO.distances(X)
    assert SO.criterion("mda", D, (0, 1, 3)) == 26 and SO.criterion("mda", D, (1, 2, 3)) == 29
    assert SO.select("mda", X, 1) == (0, 1, 3)
    assert SO.select("smea", X, 1) == (1, 2, 3)
    assert SO.criterion("smea", D, (1, 2, 3)) < SO.criterion("smea", D, (0, 1, 3))
    assert min(SO.margin(r, X, 1) for r in RULES) > 0.1


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_H0_gives_the_plain_mean(rule, dt):
    rs = np.random.RandomState(3)
    for n in (1, 2, 5, 16):
        X = rs.randn(n, 33).astype(dt)
        out, w = SO.aggregate(rule, X, 0)
        want = np.zeros(33, dt)
        for k in range(n):
            want = want + X[k]
        np.testing.assert_array_equal(out, want / dt(n))
        np.testing.assert_array_equal(w, np.full(n, dt(1) / dt(n)))


@pytest.mark.parametrize("rule", RULES)
def test_H_n_minus_1_gives_the_own_row(rule):
    rs = np.random.RandomState(4)
    for n in (1, 2, 7, 16):
        X = rs.randn(n, 9).astype(np.float32)
        X[0] *= 50                                           # far from the rest: still rank 0 = {0}
        out, w = SO.aggregate(rule, X, n - 1)
        np.testing.assert_array_equal(out, X[0])
        assert w[0] == 1 and (w[1:] == 0).all()


@pytest.mark.parametrize("rule", RULES)
def test_equal_rows_select_rank_0(rule):
    X = np.tile(np.array([[1.5, -2.0, 3.0]]), (6, 1))
    for H in range(6):
        assert SO.select(rule, X, H) == tuple(range(6 - H))
        assert all(c == 0 for c, _ in SO.scores(rule, X, H))


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("seed", range(6))
def test_up_to_H_bad_rows_get_weight_zero(rule, seed):
    rs = np.random.RandomState(100 + seed)
    n = int(rs.randint(3, 10))
    H = int(rs.randint(1, (n - 1) // 2 + 1))
    X = rs.randn(n, 20) * rs.uniform(0.1, 1, size=(n, 1))
    nb = int(rs.randint(1, H + 1))
    bad = rs.choice(n, size=nb, replace=False)
    for k in bad:
        cols = rs.choice(20, size=int(rs.randint(1, 21)), replace=False)
        X[k, cols] = rs.choice([1e30, -1e30, np.inf, -np.inf])
    out, w = SO.aggregate(rule, X, H)
    assert (w[bad] == 0).all() and np.isfinite(out).all()
    assert (w > 0).sum() == n - max(H, int(SO.flagged(X).sum()))


@pytest.mark.parametrize("rule", RULES)
def test_every_row_flagged_gives_the_own_row(rule):
    X = np.array([[np.inf, 1.0], [2.0, -np.inf], [np.inf, np.inf]])
    out, w = SO.aggregate(rule, X, 1)
    np.testing.assert_array_equal(out, X[0])
    np.testing.assert_array_equal(w, [1, 0, 0])


def test_smea_criterion_is_s_times_the_top_eigenvalue_of_the_subset_covariance():
    rs = np.random.RandomState(7)
    for n, P, H in ((4, 5, 1), (6, 3, 2), (7, 40, 3), (9, 2, 4)):
        X = rs.randn(n, P) * rs.uniform(0.2, 3, size=(n, 1))
        D = SO.distances(X)
        for c, S in SO.scores("smea", X, H):
            Y = X[list(S)]
            C = (Y - Y.mean(0)).T @ (Y - Y.mean(0)) / len(S)       # the subset's covariance
            want = len(S) * np.linalg.eigvalsh(C)[-1]
            assert abs(c - want) <= 1e-9 * max(want, 1.0), (S, c, want)
            assert abs(SO.criterion("smea", D, S) - want) <= 1e-9 * max(want, 1.0)


def test_mda_criterion_is_the_squared_diameter_by_brute_force():
    rs = np.random.RandomState(8)
    X = rs.randn(7, 6)
    for c, S in SO.scores("mda", X, 3):
        assert c == max(float(np.sum((X[a] - X[b]) ** 2)) for a in S for b in S)


def test_candidates_are_ranked_lexicographically():
    X = np.zeros((5, 1))
    X[3, 0] = np.inf
    s, cands = SO.candidates(X, 2)
    assert s == 3 and cands == [(0, 1, 2), (0, 1, 4), (0, 2, 4), (1, 2, 4)]


def test_oracle_refuses_what_the_library_refuses():
    X = np.zeros((4, 3))
    for H in (-1, 4, 5):
        for rule in RULES:
            with pytest.raises(ValueError):
                SO.aggregate(rule, X, H)
    with pytest.raises(ValueError):
        SO.aggregate("dnc", X, 1)


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enum_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "subset.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_vector_job*, int, void*) = rcmarl_subset_aggregate; (void)f;'
                   'printf("%d %d %d\\n", RCMARL_SUBSET_MDA, RCMARL_SUBSET_SMEA, RCMARL_SUBSET_MAX_FLOATS); return 0;}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_subset_aggregate(const rcmarl_vector_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "subset"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [L.SUBSET_MDA, L.SUBSET_SMEA, L.SUBSET_MAX_FLOATS] == [0, 1, 48 * 1024]
    assert 16 * 1421 <= L.SUBSET_MAX_FLOATS                  # the 16-agent team-reward net at n_in = 16
    assert ("rcmarl_subset_aggregate", ctypes.c_int, [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_subset_aggregate.argtypes == [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 rows of 100 floats, 1000 floats apart, dst far away."""
    from rcmarl import _lib as L
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = 1 << 24, 1 << 16, 1000, 100, 4, 1, L.SUBSET_SMEA
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
    dict(rule=2), dict(rule=-1), dict(H=-1), dict(H=4), dict(n_in=1, H=1),
    dict(n=48 * 1024 // 4 + 1),                                              # n_in * n over the staging bound
    dict(n_in=1, H=0, n=48 * 1024 + 1),                                      # ... by one float
    dict(dst=(1 << 16) + 4 * 2000), dict(dst=(1 << 16) + 4 * 2000 + 396), dict(dst=(1 << 16) - 4 * 99),   # overlaps rows
    dict(weights_out=(1 << 16) + 4 * 1000 + 8), dict(weights_out=(1 << 16) - 4 * 3),   # weights_out on an in-node row
    dict(weights_out=(1 << 24) + 4 * 99),                                            # ... or on the job's own dst
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    for rule in (L.SUBSET_MDA, L.SUBSET_SMEA):
        bad_job = _job(**{"rule": rule, **bad})
        for jobs in ([bad_job], [_job(dst=1 << 26, weights_out=(1 << 26) + 4096), bad_job]):
            arr = (L.VectorJob * len(jobs))(*jobs)
            assert lib.rcmarl_subset_aggregate(arr, len(arr), None) == -1             # RCMARL_ERR_ARG


def test_library_refuses_writes_on_another_jobs_ranges_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    arr = (L.VectorJob * 2)(_job(msgs=1 << 28), _job(dst=(1 << 28) + 4 * 1000))   # job 1 writes job 0's row 1
    assert lib.rcmarl_subset_aggregate(arr, 2, None) == -1
    first = dict(dst=1 << 26, weights_out=(1 << 26) + 4096)
    for second in (dict(dst=(1 << 26) + 4 * 99), dict(weights_out=(1 << 26) + 4 * 50),
                   dict(weights_out=(1 << 26) + 4096 + 12), dict(dst=(1 << 26) + 4096 - 8)):
        arr = (L.VectorJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_subset_aggregate(arr, 2, None) == -1, second
    assert lib.rcmarl_subset_aggregate(None, 1, None) == -1
    arr = (L.VectorJob * 33)(*[_job(dst=(1 << 24) + 4096 * i) for i in range(33)])
    assert lib.rcmarl_subset_aggregate(arr, 0, None) == -1
    assert lib.rcmarl_subset_aggregate(arr, 33, None) == -1


def test_rule_names_and_limits():
    from rcmarl import _lib as L
    assert L.SUBSET_RULES == {"mda": 0, "smea": 1}
    for H, n in ((0, 1), (1, 2), (15, 16), (0, 16), (7, 16)):
        assert L.check_subset_rule(H, n) is None
    for H, n in ((1, 1), (-1, 4), (4, 4), (0, 0), (0, 17)):
        with pytest.raises(L.RcmarlError):
            L.check_subset_rule(H, n)
    assert L.is_subset_rule("mda") and L.is_subset_rule("smea")
    assert not L.is_subset_rule("MDA") and not L.is_subset_rule(0) and not L.is_subset_rule("dnc")
    for name in RULES:
        assert not L.is_vector_rule(name) and not L.is_spectral_rule(name) and name not in L.AGG_RULES


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


def trainer(aggregation, H=1, labels=None, attack=None, mixing=None):
    from rcmarl.trainer import Trainer
    labels = labels or ["Cooperative"] * 4 + ["Malicious"]
    return Trainer(labels=labels, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing)


@pytest.mark.parametrize("aggregation,H,labels,attack,mixing", [
    ("mda", 4, None, None, None),                                             # H >= n_in
    ("smea", [0, 5, 0, 0, 0], None, None, None),
    (["mda", "clip", "smea", "clip", "clip"], [1, 0, -1, 0, 0], None, None, None),
    ("MDA", 1, None, None, None),
    ("smea_", 1, None, None, None),
    ("mda", 3, None, None, ("bucket", 2)),                                   # 3 bucket rows leave H = 3 >= n_out
    (["clip", "smea", "clip", "clip", "clip"], 2, None, None, ("bucket", 3)),   # 2 rows
    ("mda", 1, BYZ, ("tailored_std", 2.0), None),                            # no adaptive attack models mda / smea
    (["clip", "clip", "smea", "clip", "clip"], 1, BYZ, ("tailored_uv", 2.0), None),
    ("smea", 1, BYZ, ("pipeline_std", 2.0), None),
    (["clip", "mda", "clip", "clip", "clip"], 1, BYZ, ("pipeline_sgn", 1.0), "nnm"),
])
def test_trainer_refuses_before_any_device_work(no_device, aggregation, H, labels, attack, mixing):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(aggregation, H, labels, attack, mixing)


@pytest.mark.parametrize("aggregation,H,labels,attack,mixing", [
    ("mda", 0, None, None, None), ("smea", 3, None, None, None),
    (["mda", "trim", "krum", "smea", "clip"], [1, 1, 1, 1, 0], None, None, None),
    (["gmed", "smea", "dnc", "mkrum", "mda"], [1, 2, 1, 1, 9], BYZ, ("minmax_uv", 1.0), None),
    (["mda", "smea", "scclip", "wmsr", "clip"], [3, 2, 1, 1, 0], BYZ, ("alie", 1.0), "nnm"),
    (["smea", "mda", "dnc", "clip", "clip"], 1, BYZ, ("dissensus", 1.0), ("bucket", 2)),
    (["mda", "smea", "clip", "clip", "clip"], 1, BYZ, ("mimic", 2), [("bucket", 2), "nnm", None, None, None]),
    (["mda", "clip", "clip", "clip", "clip"], 1, BYZ, ("tailored_std", 2.0), None),   # agent 0 does not hear agent 4
    (["smea", "clip", "clip", "clip", "clip"], 1, BYZ, ("pipeline_uv", 2.0), None),   # ... nor does it here
])
def test_trainer_accepts_mda_and_smea_alone_and_mixed(no_device, aggregation, H, labels, attack, mixing):
    with pytest.raises(no_device):
        trainer(aggregation, H, labels, attack, mixing)
