"""CPU checks of nearest-neighbour mixing (rcmarl_nnm_mix, include/rcmarl.h): properties of the oracle's mixed rows and
mixing matrix (tests/nnm_oracle.py) and each consequence the header states, the enum and symbol as the header and the
bindings declare them, the library's refusals without a device, and the Trainer's refusals, acceptance and message-row
layout before it touches a device.

Selections are compared under a transformation only where they are well defined: a relative distance gap at every
row's n - H boundary above 1e-4 (nnm_oracle.margin; a tie between identical rows is exact and does not count)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import nnm_oracle as NO
import vector_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@st.composite
def case(draw, min_n=1):
    """(H, X [n, P] float64 from a seeded normal draw around a common centre, each row with its own spread)."""
    n = draw(st.integers(min_n, 16))
    H = draw(st.integers(0, n - 1))
    P = draw(st.integers(1, 40))
    rs = np.random.RandomState(draw(st.integers(0, 2 ** 31 - 1)))
    X = rs.randn(n, P) * rs.uniform(0.1, 3, size=(n, 1)) + rs.randn(P) * rs.uniform(0, 100)
    return H, X


@given(case())
@settings(max_examples=300, deadline=None)
def test_rows_of_M_are_uniform_on_N_k_and_give_the_mixed_rows(c):
    H, X = c
    n = X.shape[0]
    Y, M = NO.mix(X, H)
    sel = NO.selections(X, H)
    for k in range(n):
        on = M[k] > 0
        assert on.sum() == len(sel[k]) == n - H and M[k, k] > 0      # every distance finite here: |N_k| = n - H
        assert (M[k][on] == 1.0 / on.sum()).all() and list(np.flatnonzero(on)) == sel[k]
    np.testing.assert_allclose(Y, M @ X, rtol=1e-9, atol=1e-9 * np.abs(X).max())


@given(case(min_n=3))
@settings(max_examples=200, deadline=None)
def test_H0_every_row_is_multi_krum_at_H0_bitwise(c):
    _, X = c
    for dt in (np.float64, np.float32):
        Xd = X.astype(dt)
        Y, M = NO.mix(Xd, 0)
        want, w = VO.aggregate(Xd, 0, "mkrum")
        for k in range(X.shape[0]):
            np.testing.assert_array_equal(Y[k], want)
            np.testing.assert_array_equal(M[k], w)


@given(case())
@settings(max_examples=200, deadline=None)
def test_H_n_minus_1_passes_every_row_through_bitwise(c):
    _, X = c
    n = X.shape[0]
    for dt in (np.float64, np.float32):
        Y, M = NO.mix(X.astype(dt), n - 1)
        np.testing.assert_array_equal(Y, X.astype(dt))
        np.testing.assert_array_equal(M, np.eye(n))


POISON = (np.inf, -np.inf, 1e30, -1e30)


@given(case(min_n=2), st.data())
@settings(max_examples=200, deadline=None)
def test_rows_at_non_finite_distance_pass_through_and_are_never_mixed_in(c, data):
    """Up to H rows each at a non-finite distance from every other row (+-inf in some or all coordinates, +-1e30): each
    passes through bitwise, no finite row mixes one in, and at most that many mixed rows are not finite."""
    H, X = c
    n, P = X.shape
    n_bad = data.draw(st.integers(0, min(H, len(POISON))))
    bad = data.draw(st.permutations(range(n)))[:n_bad]
    for q, r in enumerate(bad):
        cols = np.arange(P) if data.draw(st.booleans()) or abs(POISON[q]) < np.inf else np.arange(0, P, 2)
        X[r, cols] = POISON[q]
    for dt in (np.float64, np.float32):
        Xd = X.astype(dt)
        Y, M = NO.mix(Xd, H)
        for r in bad:
            np.testing.assert_array_equal(Y[r], Xd[r])
            assert M[r, r] == 1 and (np.delete(M[:, r], r) == 0).all()
        good = [k for k in range(n) if k not in bad]
        assert np.isfinite(Y[good]).all()
        assert (~np.isfinite(Y).all(1)).sum() <= n_bad


@given(case(min_n=2), st.data())
@settings(max_examples=200, deadline=None)
def test_identical_rows_give_identical_outputs(c, data):
    H, X = c
    n = X.shape[0]
    a, b = data.draw(st.permutations(range(n)))[:2]
    X[b] = X[a]
    for dt in (np.float64, np.float32):
        Y, _ = NO.mix(X.astype(dt), H)
        np.testing.assert_array_equal(Y[a], Y[b])


@given(case(min_n=2), st.data())
@settings(max_examples=200, deadline=None)
def test_permutation_equivariant_and_selection_translation_invariant(c, data):
    H, X = c
    n = X.shape[0]
    if not NO.clear(X, H):
        return
    Y, M = NO.mix(X, H)
    pi = np.array(data.draw(st.permutations(range(n))))
    Yp, Mp = NO.mix(X[pi], H)
    np.testing.assert_array_equal(Mp, M[np.ix_(pi, pi)])
    np.testing.assert_allclose(Yp, Y[pi], rtol=1e-12, atol=1e-12 * np.abs(X).max())
    shift = np.random.RandomState(data.draw(st.integers(0, 1000))).randn(X.shape[1]) * 10
    Xs = X + shift
    if NO.clear(Xs, H):
        np.testing.assert_array_equal(NO.mix(Xs, H)[1], M)


def test_fp32_matches_fp64():
    rs = np.random.RandomState(5)
    n_cmp = 0
    for n, H in ((4, 1), (6, 2), (9, 3), (16, 7), (16, 3), (5, 0)):
        X = rs.randn(n, 700) * rs.uniform(0.2, 2, size=(n, 1)) + rs.randn(700)
        if not NO.clear(X, H):
            continue
        Y32, M32 = NO.mix(X.astype(np.float32), H)
        Y64, M64 = NO.mix(X, H)
        assert Y32.dtype == np.float32
        np.testing.assert_array_equal(M32, M64.astype(np.float32))
        np.testing.assert_allclose(Y32, Y64, rtol=1e-5, atol=1e-5)
        n_cmp += 1
    assert n_cmp >= 5


def test_hand_worked_example():
    """Points 0, 1, 3, 10 on a line, H = 1: each row mixes itself with its two nearest."""
    X = np.array([[0.0], [1.0], [3.0], [10.0]])
    Y, M = NO.mix(X, 1)
    assert NO.selections(X, 1) == [[0, 1, 2], [0, 1, 2], [0, 1, 2], [1, 2, 3]]
    np.testing.assert_allclose(Y[:, 0], [4 / 3, 4 / 3, 4 / 3, 14 / 3], rtol=1e-15)
    np.testing.assert_array_equal(M[3], [0, 1 / 3, 1 / 3, 1 / 3])
    # equal distances: the own row first, then the lower index
    Z = np.array([[0.0], [1.0], [-1.0], [1.0]])
    assert NO.selections(Z, 2) == [[0, 1], [1, 3], [0, 2], [1, 3]]
    assert NO.margin(Z, 2) == 0.0 and not NO.clear(Z, 2)
    # a repeated row: the tie is exact in any precision, so only the distances of the other rows set the gap (row 0:
    # rows 1 and 2 at 4 straddle the boundary, row 3 at 9 gives 5/9)
    R = np.array([[0.0], [2.0], [2.0], [-3.0]])
    assert NO.selections(R, 2) == [[0, 1], [1, 2], [1, 2], [0, 3]] and NO.margin(R, 2) == pytest.approx(5 / 9)


def test_oracle_refuses_what_the_library_refuses():
    X = np.zeros((4, 3))
    for H in (-1, 4, 5):
        with pytest.raises(ValueError):
            NO.mix(X, H)


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enum_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "nnm.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_vector_job*, int, void*) = rcmarl_nnm_mix; (void)f;'
                   'rcmarl_mixing_rule r = RCMARL_MIX_NNM;'
                   'printf("%d %d\\n", (int)r, RCMARL_NNM_MAX_FLOATS); return 0;}')
    exe = tmp_path / "nnm"
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_nnm_mix(const rcmarl_vector_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [L.MIX_NNM, L.NNM_MAX_FLOATS] == [0, 48 * 1024]
    assert L.MIXING_RULES == {"nnm": 0}
    assert ("rcmarl_nnm_mix", ctypes.c_int, [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_nnm_mix.argtypes == [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 rows of 100 floats, 1000 floats apart, its 4 dst rows far away at the same
    stride."""
    from rcmarl import _lib as L
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = 1 << 24, 1 << 16, 1000, 100, 4, 1, L.MIX_NNM
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
    dict(n=48 * 1024 // 4 + 1, msg_stride=48 * 1024),                         # n_in * n over the staging limit
    dict(dst=(1 << 16) + 4 * 2000),                                           # dst row 0 on in-node row 2
    dict(dst=(1 << 16) - 4 * 3000),                                           # dst row 3 on in-node row 0
    dict(dst=(1 << 16) - 4 * 2000 + 4 * 99),                                  # dst row 1 ends inside in-node row 0
    dict(msg_stride=50),                                                      # dst rows overlap each other
    dict(weights_out=(1 << 16) + 4 * 1000 + 8), dict(weights_out=(1 << 16) - 4 * 3),   # weights_out on an in-node row
    dict(weights_out=(1 << 24) + 4 * 2050),                                   # ... on the job's dst row 2
    dict(weights_out=(1 << 24) - 4 * 15),                                     # ... 16 floats reaching dst row 0
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    for jobs in ([_job(**bad)], [_job(dst=1 << 26, weights_out=(1 << 26) + 4 * 8000), _job(**bad)]):
        arr = (L.VectorJob * len(jobs))(*jobs)
        assert lib.rcmarl_nnm_mix(arr, len(arr), None) == -1                      # RCMARL_ERR_ARG


def test_library_refuses_writes_on_another_jobs_ranges_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    arr = (L.VectorJob * 2)(_job(msgs=1 << 28), _job(dst=(1 << 28) - 4 * 2000))  # job 1's dst row 3 on job 0's row 1
    assert lib.rcmarl_nnm_mix(arr, 2, None) == -1
    first = dict(dst=1 << 26, weights_out=(1 << 26) + 4 * 8000)
    for second in (dict(dst=(1 << 26) + 4 * 99), dict(dst=(1 << 26) + 4 * 8000 - 4 * 3000),   # dst rows on first's
                   dict(weights_out=(1 << 26) + 4 * 2050), dict(weights_out=(1 << 26) + 4 * 8000 + 4 * 15)):
        arr = (L.VectorJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_nnm_mix(arr, 2, None) == -1, second
    assert lib.rcmarl_nnm_mix(None, 1, None) == -1
    arr = (L.VectorJob * 33)(*[_job(dst=(1 << 24) + 4 * 4000 * i) for i in range(33)])
    assert lib.rcmarl_nnm_mix(arr, 0, None) == -1
    assert lib.rcmarl_nnm_mix(arr, 33, None) == -1


def test_mixing_names_and_limits():
    from rcmarl import _lib as L
    for H, n in ((0, 1), (1, 2), (15, 16), (0, 16), (3, 4)):
        assert L.check_mixing("nnm", H, n) == L.MIX_NNM == 0
    for H, n in ((1, 1), (-1, 4), (4, 4), (0, 0), (0, 17)):
        with pytest.raises(L.RcmarlError):
            L.check_mixing("nnm", H, n)
    for name in ("NNM", "bucketing", 0, "clip"):
        with pytest.raises(L.RcmarlError):
            L.check_mixing(name, 0, 4)
    assert "nnm" not in L.AGG_RULES and not L.is_vector_rule("nnm") and not L.is_spectral_rule("nnm")


# ------------------------------------------------------------------------------------------------ Trainer
class DeviceTouched(Exception):
    pass


@pytest.fixture
def no_device(monkeypatch):
    """Trainer construction that reaches the device fails with DeviceTouched instead."""
    import torch
    from rcmarl import _lib

    _lib.lib()

    def touched(*a, **k):
        raise DeviceTouched()
    monkeypatch.setattr(torch.cuda, "current_device", touched)
    return DeviceTouched


C5 = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
BYZ = ["Cooperative"] * 4 + ["Byzantine"]
MAL = ["Cooperative"] * 4 + ["Malicious"]


def trainer(mixing, aggregation="clip", H=1, labels=None, attack=None):
    from rcmarl.trainer import Trainer
    return Trainer(labels=labels or MAL, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing)


def built(excinfo):
    """The Trainer whose construction stopped at the device (from the frame of its __init__)."""
    tb = excinfo.tb
    while tb is not None:
        if tb.tb_frame.f_code.co_name == "__init__" and "mixing" in tb.tb_frame.f_locals:
            return tb.tb_frame.f_locals["self"]
        tb = tb.tb_next
    raise AssertionError("no Trainer frame")


@pytest.mark.parametrize("mixing,aggregation,H,labels,attack", [
    ("NNM", "clip", 1, None, None),                                           # unknown name
    (["nnm", None, "bucketing", None, None], "clip", 1, None, None),
    ([None, None, None, None, 7], "clip", 1, None, None),                     # unknown at a non-cooperative agent too
    (["nnm"] * 4, "clip", 1, None, None),                                     # wrong length
    ("nnm", "krum", [0, 0, 4, 0, 0], None, None),                             # H >= n_in
    ("nnm", "clip", 1, BYZ, ("tailored_std", 2.0)),                           # the tailored attack does not model nnm
    ([None, None, "nnm", None, None], "mkrum", 1, BYZ, ("tailored_uv", 2.0)),  # ... at one receiver of agent 4
])
def test_trainer_refuses_before_any_device_work(no_device, mixing, aggregation, H, labels, attack):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="mixing|H="):
        trainer(mixing, aggregation, H, labels, attack)


@pytest.mark.parametrize("mixing,aggregation,H,labels,attack", [
    ("nnm", "clip", 0, None, None), ("nnm", "clip", 3, None, None),
    ("nnm", ["dnc", "trim", "krum", "wmsr", "clip"], [1, 1, 1, 1, 0], None, None),
    (["nnm", None, "nnm", None, "nnm"], ["gmed", "dnc", "clip", "mkrum", "scclip"], [1, 2, 1, 1, 9], BYZ,
     ("minmax_uv", 1.0)),
    (["nnm", None, None, None, None], "clip", 1, BYZ, ("tailored_std", 2.0)),   # agent 0 does not hear agent 4
    ([None] * 5, "clip", 1, BYZ, ("tailored_std", 2.0)),
])
def test_trainer_accepts_mixing_alone_and_mixed(no_device, mixing, aggregation, H, labels, attack):
    with pytest.raises(no_device):
        trainer(mixing, aggregation, H, labels, attack)


def test_trainer_row_layout(no_device):
    """The mixed rows follow the Byzantine pair, distance-based and dnc rows; the rows of the agents that do not mix,
    and the layout without mixing, are as before."""
    with pytest.raises(no_device) as ex:
        trainer(["nnm", "nnm", None, "nnm", "nnm"], ["mkrum", "dnc", "clip", "trim", "clip"], [1, 1, 1, 1, 0], BYZ,
                ("gauss", 0.3))
    tr = built(ex)
    assert [p[:2] for p in tr.byz_pairs] == [(4, 1), (4, 2), (4, 3)]
    assert tr.vec_row == {0: 8} and tr.dnc_row == {1: 9}
    assert tr.mix_agents == [0, 1, 3] and tr.mix_row == {0: 10, 1: 14, 3: 18}       # agent 4 does not cooperate
    assert tr.mixing == ["nnm", "nnm", None, "nnm", None]
    assert tr._rule_nodes(0) == [10, 11, 12, 13] and tr._rule_nodes(3) == [18, 19, 20, 21]
    assert tr._rule_nodes(2) == tr._receiver_nodes(2) == [2, 3, 6, 0]
    assert tr._receiver_nodes(1) == [1, 2, 3, 5]
    with pytest.raises(no_device) as ex:
        trainer(None, ["mkrum", "dnc", "clip", "trim", "clip"], [1, 1, 1, 1, 0], BYZ, ("gauss", 0.3))
    tr = built(ex)
    assert tr.mix_agents == [] and tr.mix_row == {} and tr.mixing == [None] * 5
    assert tr.vec_row == {0: 8} and tr.dnc_row == {1: 9}
