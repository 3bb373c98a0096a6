"""Bit-exact fp32 restatements of the coordinate-wise kernels, and integer-valued inputs with answers in closed form,
shared by test_coord_kernel_edges_cpu.py and test_coord_kernel_edges_gpu.py.

The kernels (rcmarl_clip_mean in csrc/rollout_consensus.cu; resilient_mean_small in csrc/common.cuh, run by
rcmarl_consensus_hidden and rcmarl_team; rcmarl_attack) are fully determined: order statistics are values, sums run in
index order, and the only roundings are fp32 adds and subtracts, fminf / fmaxf, one IEEE division (the library is
built without --use_fast_math), and for ALIE an fmaf chain, an IEEE sqrtf and one more fmaf.  Each function below takes
the same operations in the same order in NumPy float32, vectorised over columns, so it matches the kernel bit for bit
on arbitrary data.  The one freedom left is the sign of a zero result: -0 and +0 are tied in every order statistic,
so which one a kernel keeps may differ; the tests compare a zero result by value.

ALIE's `mu - z * sigma` is compiled into one FFMA (read from the SASS of attack_kernel: FFMA R, -z, sigma, mu), so
alie() rounds mu - z * sigma once, with fma32.  NumPy has no fused multiply-add; fma32 forms the exact product in fp64,
adds with an error-free TwoSum and rounds to odd before the final rounding to fp32, which gives the correctly rounded
fmaf for every fp32 input whose product does not overflow fp64 (all of them).  fma32_exact is the same with Fractions.

Integer inputs (int_columns): small integers times 2^k.  Every fp32 sum the kernels take is then exact, so each answer
is one IEEE division of an exact sum (f32_round of a Fraction), computed from the header's definitions alone."""
from fractions import Fraction

import numpy as np

f32 = np.float32
F32_MAX = float(np.finfo(np.float32).max)
MAX_H = 7                                               # RCMARL_MAX_H: clip_mean's template range


# ------------------------------------------------------------------------------------------------ rounding helpers
def f32_round(x):
    """The fp32 nearest to the rational x (round half to even, subnormals, overflow to +-inf)."""
    x = Fraction(x)
    if x == 0:
        return f32(0.0)
    sign, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1                                          # 2^e <= a < 2^(e+1)
    q = max(e - 23, -149)                               # the ulp at a (subnormal spacing below 2^-126)
    m = round(a / Fraction(2) ** q)                     # Fraction.__round__: half to even
    v = m * Fraction(2) ** q
    if v > F32_MAX:
        return f32(sign * np.inf)
    return f32(sign * (float(m) * 2.0 ** q))            # exact in fp64, then exact in fp32


def fma32_exact(a, b, c):
    """fmaf(a, b, c) for fp32 scalars through exact rationals."""
    a, b, c = f32(a), f32(b), f32(c)
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return f32(np.float64(a) * np.float64(b) + np.float64(c))
    return f32_round(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def fma32(a, b, c):
    """fmaf(a, b, c) elementwise on fp32 arrays: the product is exact in fp64 (24 + 24 bits), the sum is formed with a
    TwoSum and rounded to odd (53 >= 24 + 2 bits), so the one rounding to fp32 is the correctly rounded fmaf."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)                 # s + err == p + c exactly (Knuth's TwoSum)
        odd = (s.view(np.int64) & 1) == 1
        fix = np.isfinite(s) & (err != 0) & ~odd
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


# ------------------------------------------------------------------------------------------------ rcmarl_clip_mean
def clip_mean(v, H, vec=1, paths=False, srt=None):
    """rcmarl_clip_mean over the columns of v [n, P] (fp32, own = row 0), as Track<H> computes it:
    sum in row order; small / large = the H+1 smallest / largest values; lo = fminf(small[H], own),
    hi = fmaxf(large[H], own); identity_ok = max(|small[0]|, |large[0]|) <= 16 * max(|lo|, |hi|); then either finish
    (subtract min(small[i] - lo, 0) and max(large[i] - hi, 0) for i = 0..H, in that order) or the second pass (sum of
    fmaxf(fminf(v, hi), lo) in row order); one division by n.

    vec: columns per thread.  The vector kernel (vec = 4 for H <= 1, 2 for H >= 2) takes the second pass for all of a
    thread's columns when identity_ok fails for any of them; the scalar kernel decides per column (vec = 1).
    paths=True also returns the boolean mask of columns that took the second pass; srt may pass np.sort(v, axis=0)."""
    v = np.asarray(v, np.float32)
    n, P = v.shape
    assert 0 <= H < n and P % vec == 0
    srt = np.sort(v, axis=0) if srt is None else srt
    small, large = srt[:H + 1], srt[::-1][:H + 1]
    own = v[0]
    lo, hi = np.fmin(small[H], own), np.fmax(large[H], own)
    with np.errstate(invalid="ignore", over="ignore"):       # inf - inf on outlier columns: their sum is not used
        s = np.zeros(P, np.float32)
        for k in range(n):
            s = s + v[k]
        w = np.fmax(np.abs(lo), np.abs(hi))
        m = np.fmax(np.abs(small[0]), np.abs(large[0]))
        ok = m <= f32(16) * w
        ok = np.repeat(ok.reshape(-1, vec).all(1), vec)
        r = s.copy()
        for i in range(H + 1):
            r = r - np.fmin(small[i] - lo, f32(0))
            r = r - np.fmax(large[i] - hi, f32(0))
        r2 = np.zeros(P, np.float32)
        for k in range(n):
            r2 = r2 + np.fmax(np.fmin(v[k], hi), lo)
        out = np.where(ok, r, r2) / f32(n)
    return (out, ~ok) if paths else out


def vec_width(H):
    """Columns per thread of clip_mean's vector kernel (16-byte loads for H <= 1, 8-byte for H >= 2)."""
    return 4 if H <= 1 else 2


# ------------------------------------------------------------------------------------------------ resilient_mean_small
def ranks(v):
    """rank(k) = #{m : v[m] < v[k] or (v[m] == v[k] and m < k)} over axis 0: the position of k in a stable sort."""
    order = np.argsort(v, axis=0, kind="stable")
    rank = np.empty_like(order)
    n = v.shape[0]
    np.put_along_axis(rank, order, np.broadcast_to(np.arange(n)[:, None], v.shape), axis=0)
    return rank


def resilient_mean_small(v, H, rule):
    """resilient_mean_small (csrc/common.cuh) over the columns of v [n, P] (fp32, own = row 0).  CLIP: the values of
    rank H and n-H-1, lo = fminf(., own), hi = fmaxf(., own), sum of fmaxf(fminf(v, hi), lo) in index order, / n.
    TRIM: ranks H..n-H-1 kept; WMSR: ranks min(H, below)..n-1-min(H, above) kept, with above / below counted strictly
    against own over k >= 1.  The kept values are added in index order from 0 (a dropped value never enters), then
    divided by hi - lo + 1."""
    v = np.asarray(v, np.float32)
    n, P = v.shape
    rule = {0: "clip", 1: "trim", 2: "wmsr"}.get(rule, rule)
    rank = ranks(v)
    with np.errstate(invalid="ignore", over="ignore"):
        if rule == "clip":
            assert 0 <= H < n
            srt = np.sort(v, axis=0)
            lo, hi = np.fmin(srt[H], v[0]), np.fmax(srt[n - H - 1], v[0])
            s = np.zeros(P, np.float32)
            for k in range(n):
                s = s + np.fmax(np.fmin(v[k], hi), lo)
            return s / f32(n)
        if rule == "trim":
            assert 0 <= 2 * H < n
            lo, hi = np.full(P, H), np.full(P, n - H - 1)
        elif rule == "wmsr":
            assert 0 <= H < n
            above, below = (v[1:] > v[0]).sum(0), (v[1:] < v[0]).sum(0)
            lo, hi = np.minimum(H, below), n - 1 - np.minimum(H, above)
        else:
            raise ValueError(f"unknown rule {rule!r}")
        s = np.zeros(P, np.float32)
        for k in range(n):
            s = np.where((rank[k] >= lo) & (rank[k] <= hi), s + v[k], s)
        return s / (hi - lo + 1).astype(np.float32)


# ------------------------------------------------------------------------------------------------ rcmarl_attack
def attack(v, kind, param):
    """rcmarl_attack's ALIE / IPM message over the honest rows v [n, P] (fp32, list order, repeats included):
    mu = (sum in row order) / n; ALIE: q = fmaf(v_k - mu, v_k - mu, q) in row order, sigma = sqrtf(q / n),
    m = fmaf(-z, sigma, mu); IPM: m = (-eps) * mu."""
    v = np.asarray(v, np.float32)
    n = f32(v.shape[0])
    s = np.zeros(v.shape[1:], np.float32)
    for k in range(v.shape[0]):
        s = s + v[k]
    with np.errstate(invalid="ignore", over="ignore"):
        mu = s / n
        if kind == "ipm":
            return -f32(param) * mu
        assert kind == "alie", kind
        q = np.zeros_like(s)
        for k in range(v.shape[0]):
            d = v[k] - mu
            q = fma32(d, d, q)
        sigma = np.sqrt(q / n)
        return fma32(np.full_like(mu, -f32(param)), sigma, mu)


# ------------------------------------------------------------------------------------------------ integer inputs
INT_SCALES = {"one": 1.0, "big": 2.0 ** 100, "subnormal": 2.0 ** -140}


def int_columns(rs, n, P, scale, lim=6):
    """ints [n, P] (int64) with |ints| <= lim and X = ints * scale (fp32, exact).  Column kinds, cycling: random ints
    (ties whenever n > 2 lim + 1), every row equal to own, half the rows equal to own, two values only, and zeros of
    both signs (X carries -0.0 where the sign draw is negative)."""
    ints = rs.randint(-lim, lim + 1, size=(n, P)).astype(np.int64)
    kind = np.arange(P) % 5
    ints[:, kind == 1] = ints[0, kind == 1]
    half = rs.rand(n, P) < 0.5
    ints[:, kind == 2] = np.where(half, ints[0], ints)[:, kind == 2]
    ints[:, kind == 3] = np.where(half, 1, -2)[:, kind == 3]
    zero = (kind == 4) & (rs.rand(P) < 0.5)
    ints[:, zero] = 0
    X = (ints.astype(np.float64) * scale).astype(np.float32)
    X = np.where((ints == 0) & (rs.rand(n, P) < 0.5), -0.0, X).astype(np.float32)
    assert np.array_equal(X.astype(np.float64), ints * scale)
    return ints, X


def _div(num, den, scale):
    return f32_round(Fraction(int(num)) * Fraction(scale) / int(den))


def clip_closed(ints, H, scale):
    """The clipped mean of each column of ints * scale from the definition: the values of rank H and n-H-1 of the
    column, lo / hi against own, the exact sum of the clipped values, one rounding of sum / n."""
    n = ints.shape[0]
    srt = np.sort(ints, axis=0)
    lo, hi = np.minimum(srt[H], ints[0]), np.maximum(srt[n - H - 1], ints[0])
    num = np.clip(ints, lo, hi).sum(0)
    return np.array([_div(x, n, scale) for x in num], np.float32)


def kept_closed(ints, H, rule, scale):
    """TRIM / WMSR from the definition: the exact sum of the kept values over their count, rounded once."""
    if rule == "clip":
        return clip_closed(ints, H, scale)
    n = ints.shape[0]
    rank = ranks(ints)
    if rule == "trim":
        lo, hi = np.full(ints.shape[1], H), np.full(ints.shape[1], n - H - 1)
    else:
        lo = np.minimum(H, (ints[1:] < ints[0]).sum(0))
        hi = n - 1 - np.minimum(H, (ints[1:] > ints[0]).sum(0))
    keep = (rank >= lo) & (rank <= hi)
    num = np.where(keep, ints, 0).sum(0)
    return np.array([_div(x, c, scale) for x, c in zip(num, keep.sum(0))], np.float32)


ATTACK_SCALES = {"one": 1.0, "big": 2.0 ** 50, "subnormal": 2.0 ** -140}


def symmetric_rows(rs, n, P, scale, lim=6):
    """n (even) honest rows (c + a, c - a) * scale in a shuffled order per column, 1 <= a <= 3: every fp32 sum is
    exact, mu = c * scale and every v_k - mu = +-a * scale exactly.  Returns (X, c, a)."""
    assert n % 2 == 0
    c = rs.randint(-lim, lim + 1, size=P).astype(np.int64)
    a = rs.randint(1, 4, size=P).astype(np.int64)
    sign = np.array([1, -1] * (n // 2))
    sign = np.stack([rs.permutation(sign) for _ in range(P)], 1)
    ints = c + sign * a
    X = (ints.astype(np.float64) * scale).astype(np.float32)
    assert np.array_equal(X.astype(np.float64), ints * scale)
    return X, c, a


def alie_closed(c, a, z, scale):
    """ALIE on symmetric_rows: sigma = a * scale, so m = (c - z a) * scale rounded once.  When (a * scale)^2 is below
    half the smallest subnormal (2^-150), every fmaf of the variance chain rounds to 0: sigma = 0 and m = mu."""
    out = []
    for ci, ai in zip(c, a):
        sigma = Fraction(int(ai)) * Fraction(scale)
        if sigma * sigma < Fraction(1, 2 ** 150):
            sigma = Fraction(0)
        out.append(f32_round(Fraction(int(ci)) * Fraction(scale) - Fraction(z) * sigma))
    return np.array(out, np.float32)


def ipm_closed(c, eps, scale):
    """IPM on symmetric_rows: -eps * c * scale rounded once."""
    return np.array([f32_round(-Fraction(eps) * int(ci) * Fraction(scale)) for ci in c], np.float32)
