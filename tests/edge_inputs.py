"""Inputs at the edges of the whole-message kernels (include/rcmarl.h: rcmarl_vector_aggregate, rcmarl_dnc_aggregate,
rcmarl_nnm_mix, rcmarl_bucket_mix and the attacks built on them) and their answers in closed form, shared by
test_message_kernel_edges_cpu.py (the fp64 oracles against these answers) and test_message_kernel_edges_gpu.py (the
kernels against them).

Every message is a small integer times a power of two (Case.ints * Case.scale).  Then every squared distance is an
exact integer multiple of scale^2, every fp32 sum the kernels take in index order is exact, and a mean of chosen rows
is one IEEE division (f32_mean) -- so the answers below come from the header's definitions alone, bitwise, with no
eigen-solver and no margin.  The scales 2^64 and 2^-84 put every nonzero coordinate term of a squared distance above
the fp32 range (+inf: "a distance that is not finite counts as +inf") or below half the smallest subnormal (0: the
index tie rules decide), while DnC, which centres and sums in fp64, sees the same geometry as at scale 1."""
from fractions import Fraction

import numpy as np

F32_MAX = float(np.finfo(np.float32).max)
SWEEP_P = (1, 2, 3, 31, 32, 33, 255, 256, 257, 1421)    # below, at and one past a warp and a block; the 16-agent net
EDGE_P = (1, 33, 1421)
OVER, UNDER = 2.0 ** 64, 2.0 ** -84


class Case:
    """n messages X = ints * scale (float32, exact) with the receiver's H; t: each row's coordinate along the line the
    rows lie on (x_k = c + t_k v), or None when they do not."""

    def __init__(self, name, ints, scale=1.0, H=2, t=None):
        self.name, self.ints, self.scale, self.H = name, np.asarray(ints, np.int64), float(scale), H
        assert np.abs(self.ints).max() < 2 ** 12
        self.t = None if t is None else [Fraction(int(x)) for x in t]
        self.X = (self.ints.astype(np.float64) * self.scale).astype(np.float32)
        assert np.array_equal(self.X.astype(np.float64), self.ints * self.scale)

    @property
    def n(self):
        return self.ints.shape[0]

    @property
    def P(self):
        return self.ints.shape[1]

    def __repr__(self):
        return f"{self.name}(n={self.n}, P={self.P}, H={self.H})"


# ------------------------------------------------------------------------------------------------ the cases
def _rs(P, salt):
    return np.random.RandomState(7000 + 31 * P + salt)


def identical(P, n=7, H=2):
    row = _rs(P, 1).randint(-8, 9, size=P)
    return Case(f"identical_P{P}", np.tile(row, (n, 1)), H=H, t=[0] * n)


def two_clusters(P, n=7, H=2, a_at=(1, 4)):
    """len(a_at) = H copies of a (the minority, so the furthest from the mean) and n - H copies of b."""
    rs = _rs(P, 2)
    b = rs.randint(-8, 9, size=P)
    a = b + rs.choice([-3, -2, 2, 3], size=P)
    t = [1 if k in a_at else 0 for k in range(n)]
    return Case(f"two_clusters_P{P}", np.stack([a if tk else b for tk in t]), H=H, t=t)


def line():
    """P = 1: distinct values, D_01 = D_02 (an exact distance tie), distances from x_0 whose ratios are powers of two."""
    x = [0, 1, -1, 2, -4, 8, -16]
    return Case("line_P1", np.array(x)[:, None], H=2, t=x)


def collinear(P=1421, t=(0, 3, -1, 5, -6, 2, 1)):
    rs = _rs(P, 3)
    c = rs.randint(-3, 4, size=P)
    v = rs.choice([-3, -2, -1, 1, 2, 3], size=P)
    return Case(f"collinear_P{P}", np.stack([c + tk * v for tk in t]), H=2, t=t)


def scaled(P, scale, tag):
    """Rows t_k v (v without zeros) at a scale where every fp32 squared distance overflows (OVER) or underflows (UNDER)."""
    v = _rs(P, 4).choice([-3, -2, -1, 1, 2, 3], size=P)
    t = (0, 1, -1, 2, -2, 3, -3)
    return Case(f"{tag}_P{P}", np.stack([tk * v for tk in t]), scale=scale, H=2, t=t)


def repeated(P, n=7, H=2):
    """Rows far from a central row that is listed twice (slots 2 and 5): its two copies tie exactly everywhere."""
    rs = _rs(P, 5)
    ints = rs.choice([-1, 1], size=(n, P)) * rs.randint(3, 9, size=(n, P))
    ints[2] = ints[5] = rs.randint(-1, 2, size=P)
    return Case(f"repeated_P{P}", ints, H=H)


def edge_cases():
    out = [line()]
    for P in EDGE_P:
        out += [identical(P), two_clusters(P), scaled(P, OVER, "overflow"), scaled(P, UNDER, "underflow")]
        if P > 1:
            out.append(repeated(P))
    out.append(collinear())
    return out


# ------------------------------------------------------------------------------------------------ fp32 arithmetic
def f32_mean(rows):
    """fp32 sum from 0 in row order, then one IEEE division by the count: the kernels' mean of chosen rows."""
    rows = np.asarray(rows, np.float32)
    s = np.zeros(rows.shape[1], np.float32)
    for r in rows:
        s = s + r
    return s / np.float32(len(rows))


def sqdist(case, k, l):
    """The fp32 squared distance of rows k and l as the kernels sum it: exact (a multiple of scale^2 below 2^24 of
    them), +inf when every nonzero term exceeds the fp32 range, 0 when every term is below half the smallest
    subnormal.  Anything else is not closed-form and is refused."""
    d = case.ints[k] - case.ints[l]
    units = int((d * d).sum())
    if units == 0:
        return 0.0
    u2 = case.scale * case.scale
    nz = (d * d)[d != 0]
    if nz.min() * u2 >= 2.0 ** 128:
        return np.inf
    if nz.max() * u2 < 2.0 ** -150:
        return 0.0
    assert units < 2 ** 24 and units * u2 <= F32_MAX, f"{case}: D_{k}{l} is not exact in fp32"
    return units * u2


def distances(case):
    n = case.n
    D = np.zeros((n, n))
    for k in range(n):
        for l in range(k + 1, n):
            D[k, l] = D[l, k] = sqdist(case, k, l)
    return D


# ------------------------------------------------------------------------------------------------ closed forms
def krum(case, rule):
    """(weights [n] fp32, out fp32) of krum / mkrum: score_k = the n - H - 2 smallest D_kl (exact), the m smallest
    scores (ties to the lower index); out = the fp32 mean of the selected rows in index order."""
    n, H = case.n, case.H
    D = distances(case)
    score = [sum(sorted(D[k, l] for l in range(n) if l != k)[:n - H - 2]) for k in range(n)]
    m = 1 if rule == "krum" else n - H
    sel = sorted(sorted(range(n), key=lambda k: (score[k], k))[:m])
    w = np.zeros(n, np.float32)
    w[sel] = np.float32(1) / np.float32(m)
    return w, f32_mean(case.X[sel])


def nnm(case):
    """(N_k for every k, mixed rows [n, P] fp32): l ordered by (D_kl, l != k, l), the first n - H less every l at
    +inf; mixed_k = the fp32 mean of N_k in index order."""
    n, H = case.n, case.H
    D = distances(case)
    sel = []
    for k in range(n):
        order = sorted(range(n), key=lambda l: (0.0 if l == k else D[k, l], l != k, l))[:n - H]
        sel.append(sorted(l for l in order if l == k or np.isfinite(D[k, l])))
    return sel, np.stack([f32_mean(case.X[s]) for s in sel])


def scclip(case):
    """(weights [n] fp32, out fp32) of scclip where every finite d_k = sqrt(D_k0) is exact and every c_k = tau / d_k
    is exact: out = x_0 + (sum_k c_k (x_k - x_0)) / n, each fmaf of the sum exact."""
    n, H, X = case.n, case.H, case.X
    D = distances(case)
    d = [np.float32(np.sqrt(D[k, 0])) for k in range(1, n)]
    assert all(not np.isfinite(dk) or float(dk) ** 2 == D[k + 1, 0] for k, dk in enumerate(d)), f"{case}: d_k inexact"
    tau = np.float32(0) if H >= n - 1 else sorted(d, key=lambda x: -x)[H]
    c = [np.float32(0) if not np.isfinite(dk) else (np.float32(1) if dk <= tau else tau / dk) for dk in d]
    s = np.zeros(case.P, np.float64)
    for k in range(1, n):
        if c[k - 1] != 0:
            s = s + np.float64(c[k - 1]) * (X[k].astype(np.float64) - X[0])
            assert np.array_equal(s.astype(np.float32), s), f"{case}: the scclip sum is not exact in fp32"
    out = X[0] + s.astype(np.float32) / np.float32(n)
    w = np.zeros(n, np.float32)
    sw = np.float32(0)
    for k in range(1, n):
        w[k] = c[k - 1] / np.float32(n)
        sw = np.float32(sw + w[k])
    w[0] = np.float32(1) - sw
    return w, out


def _line_scores(case):
    """(t_k - mean t)^2 of the rows along their line, exact."""
    tbar = sum(case.t) / len(case.t)
    return [(tk - tbar) ** 2 for tk in case.t]


def dnc_removed(case):
    """The H rows DnC removes from rows on a line (G of rank <= 1, lambda u_k^2 proportional to (t_k - mean t)^2):
    the H highest scores, equal scores the higher index first; with every score equal (G = 0) the H highest indices.
    The boundary must separate two different scores clearly (the kernel's scores carry the rounding of Jacobi)."""
    sc, H = _line_scores(case), case.H
    order = sorted(range(case.n), key=lambda k: (-sc[k], -k))
    if H and len(set(sc)) > 1:
        assert sc[order[H - 1]] > sc[order[H]] * (1 + Fraction(1, 1000)), f"{case}: no clear DnC boundary"
    return sorted(order[:H])


def dnc(case):
    """(weights [n] fp32, out fp32) of DnC on rows along a line: the fp32 mean of the kept rows in index order."""
    gone = set(dnc_removed(case))
    keep = [k for k in range(case.n) if k not in gone]
    w = np.zeros(case.n, np.float32)
    w[keep] = np.float32(1) / np.float32(len(keep))
    return w, f32_mean(case.X[keep])


def mimic_k0(case):
    """Init's k0 on rows along a line: the largest |t_k - mean t|, ties to the smaller k; other rows must trail it
    clearly unless they are copies of it."""
    sc = _line_scores(case)
    k0 = max(range(case.n), key=lambda k: (sc[k], -k))
    rest = [sc[k] for k in range(case.n) if case.t[k] != case.t[k0]]
    assert not rest or sc[k0] > max(rest) * (1 + Fraction(1, 1000)), f"{case}: no clear Init pick"
    return k0


def mimic(case, candidates):
    """(k*, whether z is set) of mimic with update 0 over every row as honest.  Init sets z when e_k0 is positive and
    finite in fp32 -- never for identical rows (e = 0), at OVER (+inf) or at UNDER (0); then z is along
    sign(t_k0 - mean t) v and k* is the candidate furthest that way (ties to the smaller k).  Otherwise z stays 0
    and k* is the lowest candidate."""
    cand = sorted(candidates)
    tbar = sum(case.t) / len(case.t)
    if all(tk == tbar for tk in case.t) or case.scale != 1.0:
        return cand[0], False
    k0 = mimic_k0(case)
    sgn = 1 if case.t[k0] > tbar else -1
    proj = {k: sgn * (case.t[k] - tbar) for k in cand}
    best = max(cand, key=lambda k: (proj[k], -k))
    rest = [proj[k] for k in cand if case.t[k] != case.t[best]]
    assert not rest or proj[best] - max(rest) > abs(proj[best]) / 1000, f"{case}: no clear mimic pick"
    return best, True


def gmed_overflow(case):
    """gmed where every pair of distinct rows is at +inf and one row holds the coordinate-wise median: beta is 1 / nu
    on that row and 0 elsewhere, so out is that row bitwise and w = e_k."""
    med = [k for k in range(case.n) if np.array_equal(case.X[k], np.median(case.X.astype(np.float64), 0))]
    assert len(med) == 1, f"{case}: the median is not one row"
    w = np.zeros(case.n, np.float32)
    w[med[0]] = 1
    return w, case.X[med[0]].copy()


def minmax_sgn_p1(values):
    """P = 1, d = -sign(mu): gamma = max_k |mu + g d - v_k| <= max - min solved exactly, gamma = mu - min (mu > 0) or
    max - mu (mu < 0), so the message is the honest extreme on the side away from the mean's sign."""
    v = [Fraction(int(x)) for x in values]
    mu = sum(v) / len(v)
    assert mu != 0 and mu.denominator == 1
    g = mu - min(v) if mu > 0 else max(v) - mu
    return float(g), float(min(v) if mu > 0 else max(v))


def minsum_sgn_p1(values):
    """P = 1, d = -sign(mu), an integer mean (so sum_k b_k = 0 exactly): n g^2 + sum_k e_k = c, gamma = the header's
    sqrtf(n (c - sum e)) / n (one sqrtf of an exact integer, one division) and its exact value sqrt((c - sum e) / n)."""
    v = [int(x) for x in values]
    n = len(v)
    assert sum(v) % n == 0 and sum(v) != 0
    mu = sum(v) // n
    c = max(sum((v[k] - v[l]) ** 2 for l in range(n) if l != k) for k in range(n))
    m = c - sum((x - mu) ** 2 for x in v)
    assert 0 < n * m < 2 ** 24
    g32 = np.float32(np.sqrt(np.float32(n * m))) / np.float32(n)
    d = -1.0 if mu > 0 else 1.0
    return g32, float(np.sqrt(m / n)), np.float32(np.float32(mu) + g32 * np.float32(d))


def dissensus(case, n_byz, eps):
    """x_0 - (eps / n_byz) sum_k (v_k - x_0) over every row as honest (row 0 the receiver), exact in fp32 for the
    dyadic eps / n_byz used here."""
    X = case.X.astype(np.float64)
    c = eps / n_byz
    assert np.float32(c) == c and (c * 2 ** 8).is_integer()
    want = X[0] - c * (X - X[0]).sum(0)
    assert np.array_equal(want.astype(np.float32), want), f"{case}: dissensus not exact in fp32"
    return want.astype(np.float32)
