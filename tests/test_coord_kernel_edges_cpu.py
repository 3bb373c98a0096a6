"""The coordinate-wise kernels without a GPU:

- the sorting networks compiled into clip_mean (SortNet<N> in csrc/rollout_consensus.cu), parsed from the source: each
  sorts every 0-1 input and equals tools/gen_sortnets.py's list;
- Track<H>'s push, push2 and push_group8 restated on those networks, driven as the vector and scalar kernels drive
  them: they keep the H+1 smallest and largest values for every H in 0..7, on every sequence over {0, 1, 2} up to
  n = 10 and on random sequences at every n mod 8;
- the fp32 restatements of tests/coord_oracle.py against the closed forms bitwise on integer inputs (scales 1, 2^100,
  2^-140 (subnormal), 2^50), and against the fp64 oracles (O.resilient_aggregation, agg_oracle, attack_oracle) within
  the rounding bound of the kernels' fp32 sums on random data;
- fma32 against exact rationals, and f32_round at ties and subnormals;
- every refusal of rcmarl_clip_mean, rcmarl_consensus_hidden, rcmarl_team and rcmarl_attack: on a machine without a
  device a refused call returns RCMARL_ERR_ARG, while a valid call reaches its launch and fails with another code, so
  each refusal is told apart from a launch without running anything.  Those tests skip where a device is present, so a
  negative in-node never goes near a GPU."""
import ast
import ctypes as C
import itertools
import os
import re
from fractions import Fraction

import numpy as np
import pytest

import agg_oracle as AO
import attack_oracle as AT
import coord_oracle as CO
from oracle import rpbcac_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


# ------------------------------------------------------------------------------------------------ sorting networks
def compiled_nets():
    """{N: [(i, j), ...]} of every SortNet<N> specialisation in csrc/rollout_consensus.cu, in source order."""
    src = open(os.path.join(ROOT, "resilient-consensus-based-marl_b200", "csrc", "rollout_consensus.cu")).read()
    nets = {}
    for m in re.finditer(r"template <> struct SortNet<(\d+)> \{(.*?)\} \};", src):
        nets[int(m.group(1))] = [(int(i), int(j)) for i, j in
                                 re.findall(r"cswap<ASC>\(a\[(\d+)\], a\[(\d+)\]\);", m.group(2))]
    return nets


def generator_nets():
    """NETS of tools/gen_sortnets.py, read without running the script."""
    tree = ast.parse(open(os.path.join(ROOT, "tools", "gen_sortnets.py")).read())
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "NETS" for t in node.targets):
            return ast.literal_eval(node.value)
    raise AssertionError("NETS not found")


NETS = compiled_nets()


def test_every_network_is_compiled_and_equals_the_generator():
    assert sorted(NETS) == list(range(1, 9))
    assert NETS[1] == []
    gen = generator_nets()
    assert sorted(gen) == list(range(2, 9))
    for N in range(2, 9):
        assert NETS[N] == [tuple(c) for c in gen[N]], N
    assert [len(NETS[N]) for N in range(2, 9)] == [1, 3, 5, 9, 12, 16, 19]    # optimal comparator counts


@pytest.mark.parametrize("N", range(1, 9))
def test_every_network_sorts_every_zero_one_input(N):
    """0-1 principle: a comparator network that sorts all 2^N 0-1 inputs sorts every input."""
    a = np.array(list(itertools.product([0, 1], repeat=N)), np.int8).T        # [N, 2^N]
    for i, j in NETS[N]:
        assert 0 <= i < j < N
        a[i], a[j] = np.minimum(a[i], a[j]), np.maximum(a[i], a[j])
    assert (np.diff(a, axis=0) >= 0).all()


# ------------------------------------------------------------------------------------------------ Track<H> restated
def cswap(a, i, j, asc):
    lo, hi = np.minimum(a[i], a[j]), np.maximum(a[i], a[j])
    a[i], a[j] = (lo, hi) if asc else (hi, lo)


def sortnet(a, asc):
    for i, j in NETS[len(a)]:
        cswap(a, i, j, asc)


class Track:
    """Track<H> over many columns at once (numpy rows of the column vectors), as csrc/rollout_consensus.cu writes it."""

    def __init__(self, H, P):
        self.H = H
        self.small = [np.full(P, np.inf) for _ in range(H + 1)]
        self.large = [np.full(P, -np.inf) for _ in range(H + 1)]

    def push(self, v):
        H, c = self.H, v
        for i in range(H):
            lo, c = np.minimum(self.small[i], c), np.maximum(self.small[i], c)
            self.small[i] = lo
        self.small[H] = np.minimum(self.small[H], c)
        c = v
        for i in range(H):
            hi, c = np.maximum(self.large[i], c), np.minimum(self.large[i], c)
            self.large[i] = hi
        self.large[H] = np.maximum(self.large[H], c)

    def push2(self, a, b):
        assert self.H == 1
        lo, hi = np.minimum(a, b), np.maximum(a, b)
        m = np.maximum(self.small[0], lo)
        self.small[0] = np.minimum(self.small[0], lo)
        self.small[1] = np.minimum(np.minimum(self.small[1], hi), m)
        w = np.minimum(self.large[0], hi)
        self.large[0] = np.maximum(self.large[0], hi)
        self.large[1] = np.maximum(np.maximum(self.large[1], lo), w)

    def push_group8(self, g):
        K = self.H + 1
        g = list(g)
        sortnet(g, True)
        for i in range(K):
            self.small[i] = np.minimum(self.small[i], g[K - 1 - i])
        sortnet(self.small, True)
        for i in range(K):
            self.large[i] = np.maximum(self.large[i], g[8 - K + i])
        sortnet(self.large, False)


def vector_track(v, H):
    """The row loop of clip_mean_vec_kernel: groups of 8 rows (push_group8 for H >= 2, push2 pairs for H == 1, push
    for H == 0), then the n mod 8 remaining rows one at a time."""
    t, n, k = Track(H, v.shape[1]), v.shape[0], 0
    while k + 8 <= n:
        if H >= 2:
            t.push_group8(v[k:k + 8])
        elif H == 1:
            for u in range(0, 8, 2):
                t.push2(v[k + u], v[k + u + 1])
        else:
            for u in range(8):
                t.push(v[k + u])
        k += 8
    for kk in range(k, n):
        t.push(v[kk])
    return t


def scalar_track(v, H):
    t = Track(H, v.shape[1])
    for row in v:
        t.push(row)
    return t


def check_track(t, v, H, tag):
    srt = np.sort(v, axis=0)
    for i in range(H + 1):
        np.testing.assert_array_equal(t.small[i], srt[i], err_msg=f"{tag} small[{i}]")
        np.testing.assert_array_equal(t.large[i], srt[-1 - i], err_msg=f"{tag} large[{i}]")


@pytest.mark.parametrize("H", range(0, 8))
def test_track_keeps_the_extremes_on_every_sequence_over_three_values(H):
    for n in range(H + 1, 11):
        v = np.array(list(itertools.product([0, 1, 2], repeat=n)), np.float64).T   # [n, 3^n]: every sequence
        check_track(vector_track(v, H), v, H, f"vector H={H} n={n}")
        check_track(scalar_track(v, H), v, H, f"scalar H={H} n={n}")


@pytest.mark.parametrize("H", range(0, 8))
def test_track_keeps_the_extremes_at_every_remainder(H):
    rs = np.random.RandomState(4100 + H)
    for n in range(max(H + 1, 8), 33):
        v = rs.randint(0, 4, size=(n, 3000)).astype(np.float64)
        v[:, :1000] = rs.randn(n, 1000)
        check_track(vector_track(v, H), v, H, f"vector H={H} n={n}")
        check_track(scalar_track(v, H), v, H, f"scalar H={H} n={n}")


# ------------------------------------------------------------------------------------------------ rounding helpers
def test_f32_round_at_ties_subnormals_and_overflow():
    one = Fraction(1)
    assert CO.f32_round(one + Fraction(1, 2 ** 24)) == np.float32(1)                          # tie: to even
    assert CO.f32_round(one + Fraction(3, 2 ** 24)) == np.float32(1 + 2 ** -22)              # tie: to even (up)
    assert CO.f32_round(one + Fraction(1, 2 ** 24) + Fraction(1, 2 ** 80)) == np.float32(1 + 2 ** -23)
    assert CO.f32_round(Fraction(1, 2 ** 150)) == 0                                         # half the least subnormal
    assert CO.f32_round(Fraction(3, 2 ** 151)) == np.float32(2.0 ** -149)
    assert CO.f32_round(Fraction(3, 2 ** 150)) == np.float32(2.0 ** -148)                   # tie: to even
    assert CO.f32_round(-Fraction(5, 2 ** 149) / 3) == -np.float32(2.0 ** -149) * 2
    assert CO.f32_round(Fraction(2 ** 128)) == np.inf and CO.f32_round(-Fraction(2 ** 128)) == -np.inf
    rs = np.random.RandomState(4200)
    for x in np.concatenate([rs.randn(300) * 10.0 ** rs.randint(-45, 38, 300), rs.randn(100) * 1e-41]):
        assert CO.f32_round(Fraction(float(x))) == np.float32(x)                                # fp64 -> fp32


def test_fma32_is_the_correctly_rounded_fmaf():
    rs = np.random.RandomState(4300)
    a = (rs.randn(4000) * 10.0 ** rs.randint(-20, 20, 4000)).astype(np.float32)
    b = (rs.randn(4000) * 10.0 ** rs.randint(-20, 20, 4000)).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + rs.randn(4000) * 2.0 ** -rs.randint(10, 40, 4000))).astype(np.float32)
    c[:1000] = (rs.randn(1000) * 10.0 ** rs.randint(-40, 37, 1000)).astype(np.float32)
    x = np.float32(1 + 2 ** -12)                    # x * x = 1 + 2^-11 + 2^-24: an exact fp32 tie
    edge = [(x, x, 0.0), (x, x, 2.0 ** -60), (x, x, -2.0 ** -60), (-x, x, 2.0 ** -60),
            (2.0 ** -75, 2.0 ** -75, 0.0), (2.0 ** -75, 3 * 2.0 ** -75, 2.0 ** -149), (3e-30, 5e-20, -1e-45),
            (1e20, 1e20, -1e38), (3e38, 2.0, -3.4e38)]
    a = np.concatenate([a, np.float32([e[0] for e in edge])])
    b = np.concatenate([b, np.float32([e[1] for e in edge])])
    c = np.concatenate([c, np.float32([e[2] for e in edge])])
    got = CO.fma32(a, b, c)
    want = np.array([CO.fma32_exact(x_, y_, z_) for x_, y_, z_ in zip(a, b, c)], np.float32)
    np.testing.assert_array_equal(got, want)
    assert got[-9] == np.float32(1 + 2 ** -11) and got[-8] == np.float32(1 + 2 ** -11 + 2 ** -23)   # the tie, alone
    assert got[-7] == np.float32(1 + 2 ** -11)                                            # and nudged either way


# ------------------------------------------------------------------------------------------------ closed forms
def _ns(H):
    return sorted({H + 1, 7, 8, 9, 15, 16, 17, 24, 25} - set(range(H + 1)))


@pytest.mark.parametrize("scale", CO.INT_SCALES, ids=list(CO.INT_SCALES))
@pytest.mark.parametrize("H", range(0, 8))
def test_clip_mean_restatement_matches_the_closed_form(H, scale):
    """Integer inputs: both paths (identity and second pass) give the exact sum, so every grouping of the identity
    decision gives the one IEEE division of the closed form."""
    rs = np.random.RandomState(4400 + H)
    for n in _ns(H):
        ints, X = CO.int_columns(rs, n, 260, CO.INT_SCALES[scale])
        want = CO.clip_closed(ints, H, CO.INT_SCALES[scale])
        for vec in (1, 2, 4):
            got = CO.clip_mean(X, H, vec)
            np.testing.assert_array_equal(got, want, err_msg=f"H={H} n={n} vec={vec}")
        if scale == "subnormal":
            assert (np.abs(want[want != 0]) < 2.0 ** -126).all()
            assert (want != 0).sum() > 100


@pytest.mark.parametrize("scale", CO.INT_SCALES, ids=list(CO.INT_SCALES))
@pytest.mark.parametrize("rule", AO.RULES)
def test_resilient_mean_small_restatement_matches_the_closed_form(rule, scale):
    rs = np.random.RandomState(4500)
    for n in range(1, 17):
        for H in range(0, n):
            if rule == "trim" and 2 * H >= n:
                continue
            ints, X = CO.int_columns(rs, n, 60, CO.INT_SCALES[scale])
            np.testing.assert_array_equal(CO.resilient_mean_small(X, H, rule), CO.kept_closed(ints, H, rule, CO.INT_SCALES[scale]),
                                          err_msg=f"{rule} n={n} H={H}")


@pytest.mark.parametrize("scale", CO.ATTACK_SCALES, ids=list(CO.ATTACK_SCALES))
def test_attack_restatement_matches_the_closed_form(scale):
    rs = np.random.RandomState(4600)
    s = CO.ATTACK_SCALES[scale]
    for n in (2, 4, 6, 16):
        X, c, a = CO.symmetric_rows(rs, n, 300, s)
        for z in (0.0, 1.0, -1.0, 2.0, -2.0, 0.5, 1.5):
            np.testing.assert_array_equal(CO.attack(X, "alie", z), CO.alie_closed(c, a, z, s), err_msg=f"n={n} z={z}")
            np.testing.assert_array_equal(CO.attack(X, "ipm", z), CO.ipm_closed(c, z, s), err_msg=f"n={n} eps={z}")


# ------------------------------------------------------------------------------------------------ fp64 oracles
def sum_bound(n, H, v):
    """|fp32 - exact| for a mean of n values built from n + 2(H + 1) fp32 adds of terms no larger than 2 max|v|, and
    one division: (n + 2H + 3) u (n + 4H + 4) max|v| / n + u max|v|."""
    m = float(np.abs(v).max(initial=0.0))
    return (n + 2 * H + 3) * U * (n + 4 * H + 4) * m / n + U * m


def random_columns(rs, n, P, outliers=0):
    X = (rs.randn(n, P) * rs.uniform(0.1, 3.0, size=(n, 1))).astype(np.float32)
    X[:, ::7] = rs.randint(-2, 3, size=(n, X[:, ::7].shape[1]))            # ties
    X[:, 3::11] = X[0, 3::11]                                                # equal to own
    for k in range(outliers):                                                # <= H outliers in non-own rows
        rows = rs.randint(1, n, size=P)
        X[rows, np.arange(P)] = rs.choice([1e8, -1e8, 1e30, -1e30], size=P) * (rs.rand(P) < 0.3)
    return X


@pytest.mark.parametrize("H", range(0, 8))
def test_clip_mean_restatement_against_the_fp64_oracle(H):
    rs = np.random.RandomState(4700 + H)
    for n in _ns(H) + [64, 65]:
        for outliers in (0, H):
            X = random_columns(rs, n, 400, outliers)
            want = O.resilient_aggregation(X.astype(np.float64), H)
            honest = np.where(np.abs(X) < 1e7, X, 0)
            for vec in (1, 2, 4):
                got = CO.clip_mean(X, H, vec)
                # the identity path only runs while every extreme is within 16x of the (honest) clipping window
                np.testing.assert_allclose(got, want, rtol=0, atol=16 * sum_bound(n, H, honest), err_msg=f"n={n} vec={vec}")
            if outliers:
                _, second = CO.clip_mean(X, H, 1, paths=True)
                assert second.any() and not second.all()


@pytest.mark.parametrize("rule", AO.RULES)
def test_resilient_mean_small_restatement_against_agg_oracle(rule):
    rs = np.random.RandomState(4800)
    for n in range(1, 17):
        for H in range(0, n):
            if rule == "trim" and 2 * H >= n:
                continue
            X = random_columns(rs, n, 200)
            got = CO.resilient_mean_small(X, H, rule)
            want = AO.resilient_aggregation(X.astype(np.float64), H, rule)
            np.testing.assert_allclose(got, want, rtol=0, atol=sum_bound(n, 0, X), err_msg=f"{rule} n={n} H={H}")


def test_resilient_mean_small_drops_infinities_exactly():
    """<= H values of +-inf or +-1e30 in non-own rows: every rule stays finite and within the honest rounding bound of
    the fp64 oracle, and TRIM / WMSR give the same bits when each infinity becomes +-3e38 (the ranks do not change, and
    a dropped value never enters the sum)."""
    rs = np.random.RandomState(4900)
    for n in range(3, 17):
        for H in range(1, (n - 1) // 2 + 1):
            X = random_columns(rs, n, 300)
            bad = np.zeros_like(X, bool)
            for k in range(H):
                bad[rs.randint(1, n, size=300), np.arange(300)] = True
            Xb = np.where(bad, rs.choice([np.inf, -np.inf, 1e30, -1e30], size=X.shape).astype(np.float32), X)
            Xf = np.where(np.isinf(Xb), np.sign(Xb) * 3e38, Xb).astype(np.float32)
            for rule in AO.RULES:
                got = CO.resilient_mean_small(Xb, H, rule)
                assert np.isfinite(got).all(), (rule, n, H)
                np.testing.assert_allclose(got, AO.resilient_aggregation(Xb.astype(np.float64), H, rule), rtol=0,
                                           atol=sum_bound(n, 0, X), err_msg=rule)
                if rule != "clip":
                    np.testing.assert_array_equal(got, CO.resilient_mean_small(Xf, H, rule), err_msg=rule)


def test_attack_restatement_against_attack_oracle():
    rs = np.random.RandomState(5000)
    for n in range(1, 17):
        X = random_columns(rs, n, 500)
        for kind, param in (("alie", 1.5), ("alie", -0.7), ("ipm", 0.5), ("ipm", -3.0)):
            got = CO.attack(X, kind, param)
            want = AT.craft(X.astype(np.float64), kind, param)
            m = float(np.abs(X).max())
            np.testing.assert_allclose(got, want, rtol=0, atol=4 * (n + 4) * U * m * (1 + abs(param)),
                                       err_msg=f"{kind} n={n}")


# ------------------------------------------------------------------------------------------------ refusals
@pytest.fixture(scope="module")
def abi():
    """The library on a machine without a CUDA device (the valid calls below would launch on fake addresses)."""
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("refusals are told from launches only without a device")
    from rcmarl import _lib
    return _lib


ERR_ARG = -1
A, B, D, W, T = 1 << 20, 1 << 24, 1 << 26, 1 << 28, 1 << 30          # made-up device addresses


def launched(code):
    """A call that passed every check and failed at its launch (no device here)."""
    return code not in (0, ERR_ARG)


CLIP_BAD = [dict(vals=None), dict(out=None), dict(n=0), dict(n=-1), dict(P=-1), dict(row_stride=99),
            dict(H=-1), dict(H=8, n=20), dict(H=16), dict(H=4, n=4), dict(H=1, n=1)]


@pytest.mark.parametrize("bad", CLIP_BAD, ids=[str(b) for b in CLIP_BAD])
def test_clip_mean_refusals(abi, bad):
    a = dict(vals=A, n=16, P=100, row_stride=100, H=3, out=B)
    lib = abi.lib()
    assert launched(lib.rcmarl_clip_mean(a["vals"], a["n"], a["P"], a["row_stride"], a["H"], a["out"], None))
    a.update(bad)
    assert lib.rcmarl_clip_mean(a["vals"], a["n"], a["P"], a["row_stride"], a["H"], a["out"], None) == ERR_ARG


def test_clip_mean_at_the_bounds_reaches_the_launch(abi):
    lib = abi.lib()
    assert lib.rcmarl_clip_mean(A, 16, 0, 0, 3, B, None) == 0                  # P == 0: nothing to do
    for n, P, stride, H in ((8, 100, 100, 7), (1, 1, 1, 0), (129, 5, 7, 0), (17, 1, 1, 7)):
        assert launched(lib.rcmarl_clip_mean(A, n, P, stride, H, B, None)), (n, P, stride, H)


def consensus_job(abi, **kw):
    j = abi.ConsensusJob()
    j.dst, j.msgs, j.msg_stride, j.n_hidden, j.n_in, j.H, j.rule = D, A, 1000, 500, 4, 1, 0
    for k in range(4):
        j.in_nodes[k] = k
    for k, v in kw.items():
        if k == "in_nodes":
            for i, x in enumerate(v):
                j.in_nodes[i] = x
        else:
            setattr(j, k, v)
    return j


CONSENSUS_BAD = [dict(dst=None), dict(msgs=None), dict(n_hidden=0), dict(n_hidden=-3), dict(n_in=0), dict(n_in=17),
                 dict(H=-1), dict(H=4), dict(rule=3), dict(rule=-1), dict(rule=1, H=2),
                 dict(in_nodes=[-1, 1, 2, 3]), dict(in_nodes=[0, 1, 2, -5]), dict(in_nodes=[0, -2 ** 31, 2, 3]),
                 dict(n_in=16, H=7, in_nodes=list(range(15)) + [-1])]


@pytest.mark.parametrize("bad", CONSENSUS_BAD, ids=[str(b) for b in CONSENSUS_BAD])
def test_consensus_hidden_refusals(abi, bad):
    lib = abi.lib()
    good = consensus_job(abi, dst=W)
    for jobs in ([consensus_job(abi, **bad)], [good, consensus_job(abi, **bad)]):
        arr = (abi.ConsensusJob * len(jobs))(*jobs)
        assert lib.rcmarl_consensus_hidden(arr, len(arr), None) == ERR_ARG


def test_consensus_hidden_valid_calls_reach_the_launch(abi):
    """Every rule at its largest H, 16 in-nodes with repeats and in-node 0 only, a negative in-node beyond n_in (not
    read), and the job counts at their bounds."""
    lib = abi.lib()
    for kw in (dict(), dict(n_in=16, H=15, in_nodes=[0] * 16), dict(n_in=16, H=7, rule=1), dict(n_in=16, H=15, rule=2),
               dict(n_in=2, in_nodes=[3, 3, -1, -1]), dict(n_hidden=1, n_in=1, H=0)):
        arr = (abi.ConsensusJob * 1)(consensus_job(abi, **kw))
        assert launched(lib.rcmarl_consensus_hidden(arr, 1, None)), kw
    arr = (abi.ConsensusJob * 33)(*[consensus_job(abi, dst=D + 4000 * i) for i in range(33)])
    assert launched(lib.rcmarl_consensus_hidden(arr, 32, None))
    assert lib.rcmarl_consensus_hidden(arr, 33, None) == ERR_ARG
    assert lib.rcmarl_consensus_hidden(arr, 0, None) == ERR_ARG
    assert lib.rcmarl_consensus_hidden(None, 1, None) == ERR_ARG


def rows(abi, **kw):
    r = abi.Rows()
    r.sa, r.ns, r.r, r.row_begin, r.n_rows, r.time_idx, r.n_envs, r.n_agents = A, B, D, 0, 300, None, 1, 5
    for k, v in kw.items():
        setattr(r, k, v)
    return r


def team_job(abi, **kw):
    j = abi.TeamJob()
    j.w, j.msgs, j.msg_stride, j.sums, j.agg_out, j.agg_in = W, T, 800, None, W + 40000, None
    j.kind, j.n_in, j.H, j.rule = 0, 4, 1, 0
    for k in range(4):
        j.in_nodes[k] = k
    for k, v in kw.items():
        if k == "in_nodes":
            for i, x in enumerate(v):
                j.in_nodes[i] = x
        else:
            setattr(j, k, v)
    return j


TEAM_BAD = [dict(w=None), dict(kind=3), dict(kind=-1), dict(agg_out=None), dict(msgs=None), dict(n_in=0),
            dict(n_in=17), dict(H=-1), dict(H=4), dict(rule=3), dict(rule=-1), dict(rule=1, H=2),
            dict(in_nodes=[0, -1, 2, 3]), dict(in_nodes=[0, 1, 2, -7]), dict(n_in=16, H=3, in_nodes=[2] * 15 + [-1])]
ROWS_BAD = [dict(sa=None), dict(ns=None), dict(r=None), dict(n_rows=-1), dict(n_envs=0), dict(n_envs=-2),
            dict(n_agents=4), dict(n_agents=6), dict(time_idx=T + 4000, n_envs=7)]


@pytest.mark.parametrize("bad", TEAM_BAD, ids=[str(b) for b in TEAM_BAD])
def test_team_job_refusals(abi, bad):
    lib = abi.lib()
    R = rows(abi)
    good = team_job(abi, agg_out=W + 80000)
    for jobs in ([team_job(abi, **bad)], [good, team_job(abi, **bad)], [team_job(abi, **bad), good]):
        arr = (abi.TeamJob * len(jobs))(*jobs)
        assert lib.rcmarl_team(C.byref(R), arr, len(arr), None, 0, None) == ERR_ARG


@pytest.mark.parametrize("bad", ROWS_BAD, ids=[str(b) for b in ROWS_BAD])
def test_team_rows_refusals(abi, bad):
    lib = abi.lib()
    arr = (abi.TeamJob * 1)(team_job(abi))
    assert launched(lib.rcmarl_team(C.byref(rows(abi)), arr, 1, None, 0, None))
    assert lib.rcmarl_team(C.byref(rows(abi, **bad)), arr, 1, None, 0, None) == ERR_ARG


def test_team_valid_calls_reach_the_launch(abi):
    """agg_in jobs read no in-node (a negative one is not refused there), every MAXN bound, 16 agents, gathered rows,
    n_rows = 0; a sums job without a workspace is RCMARL_ERR_WORKSPACE, not a refusal of its arguments."""
    lib = abi.lib()
    for rkw, jkw in ((dict(), dict(agg_in=T + 80000, in_nodes=[-1] * 4, n_in=0, H=-1, rule=9, msgs=None)),
                     (dict(), dict(n_in=1, H=0, in_nodes=[5])), (dict(), dict(n_in=5, H=4, rule=2)),
                     (dict(), dict(n_in=8, H=3, rule=1)), (dict(), dict(n_in=9, H=8)),
                     (dict(), dict(n_in=16, H=15, rule=2, in_nodes=[0] * 16)),
                     (dict(n_agents=16), dict(kind=1)), (dict(n_agents=16), dict(kind=2)),
                     (dict(time_idx=T + 4000, n_envs=3, n_rows=300), dict())):
        arr = (abi.TeamJob * 1)(team_job(abi, **jkw))
        assert launched(lib.rcmarl_team(C.byref(rows(abi, **rkw)), arr, 1, None, 0, None)), (rkw, jkw)
    arr = (abi.TeamJob * 1)(team_job(abi, sums=W + 90000))
    assert lib.rcmarl_team(C.byref(rows(abi)), arr, 1, None, 0, None) == -2              # RCMARL_ERR_WORKSPACE
    arr = (abi.TeamJob * 33)(*[team_job(abi, agg_out=W + 4000 * i) for i in range(33)])
    assert launched(lib.rcmarl_team(C.byref(rows(abi)), arr, 32, None, 0, None))
    for n in (0, 33):
        assert lib.rcmarl_team(C.byref(rows(abi)), arr, n, None, 0, None) == ERR_ARG
    assert lib.rcmarl_team(C.byref(rows(abi)), None, 1, None, 0, None) == ERR_ARG
    assert lib.rcmarl_team(None, arr, 1, None, 0, None) == ERR_ARG


def attack_job(abi, **kw):
    j = abi.AttackJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_honest, j.kind, j.param = D, A, 1500, 1421, 3, 0, 1.5
    j.seed, j.attacker, j.receiver, j.round, j.epoch = 7, 255, 255, 1, 2
    for k in range(3):
        j.honest[k] = k
    for k, v in kw.items():
        if k == "honest":
            for i, x in enumerate(v):
                j.honest[i] = x
        else:
            setattr(j, k, v)
    return j


ATTACK_BAD = [dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-1), dict(n_honest=0), dict(n_honest=17),
              dict(honest=[0, -1, 2]), dict(kind=3), dict(kind=-1), dict(param=float("inf")), dict(param=float("nan")),
              dict(kind=2, param=-0.5), dict(attacker=256), dict(receiver=256)]


@pytest.mark.parametrize("bad", ATTACK_BAD, ids=[str(b) for b in ATTACK_BAD])
def test_attack_refusals(abi, bad):
    lib = abi.lib()
    for jobs in ([attack_job(abi, **bad)], [attack_job(abi, dst=W), attack_job(abi, **bad)]):
        arr = (abi.AttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_attack(arr, len(arr), None) == ERR_ARG


def test_attack_valid_calls_reach_the_launch(abi):
    lib = abi.lib()
    for kw in (dict(), dict(kind=1, param=-3.0), dict(kind=2, param=0.0), dict(n_honest=16, honest=[4] * 16),
               dict(n=1, n_honest=1, attacker=0, receiver=0)):
        arr = (abi.AttackJob * 1)(attack_job(abi, **kw))
        assert launched(lib.rcmarl_attack(arr, 1, None)), kw
    arr = (abi.AttackJob * 33)(*[attack_job(abi, dst=D + 8000 * i) for i in range(33)])
    assert launched(lib.rcmarl_attack(arr, 32, None))
    for n in (0, 33):
        assert lib.rcmarl_attack(arr, n, None) == ERR_ARG
    assert lib.rcmarl_attack(None, 1, None) == ERR_ARG
