"""The coordinate-wise kernels bit for bit against the fp32 restatements of tests/coord_oracle.py, at the edges of
their ABI:

- rcmarl_clip_mean for every H in 0..7, n in {H+1, 7, 8, 9, 15, 16, 17, 24, 25, 64, 65, 129}, P in {1, 2, 3, 4, 5, 7,
  8, 255, 256, 257, 1024, 1025}, once aligned (the vector kernel wherever P allows it) and once with the input at a
  1-float offset, an odd row stride and an offset output (the scalar kernel); random columns with ties, columns equal
  to own and outlier columns holding <= H entries of 1e8, +-1e30 or +-inf (so both the single-pass identity and the
  second pass run), integer columns at 2^0, 2^100 and 2^-140 (subnormal results) against their closed forms, and the
  C5 shape (64 x 1 048 576) for every H;
- rcmarl_consensus_hidden, launches of 32 mixed-rule jobs: every rule x n_in 1..16 x every H the rule allows x
  n_hidden in {1, 255, 256, 257, 1400}, repeated in-nodes, an odd msg_stride, messages at an odd float offset, and
  rows of +-inf / +-1e30 in at most H slots;
- rcmarl_team with agg_out-only jobs whose neighbour heads have W3 = 0: every estimate is then exactly its b3, so
  agg_out is exact on every row; every rule x n_in 1..16 (the MAXN = 4 / 8 / 16 instantiations and both bounds of
  each), 5 and 16 agents, S / SA / NS inputs in one call, contiguous and gathered rows, and row counts that leave the
  second row of a thread's pair dead;
- rcmarl_attack: ALIE and IPM bitwise at n_honest 1..16 with repeats, P in {1, 255, 256, 257, 1421}, 32 jobs per
  launch, on symmetric integer rows against their closed forms, and GAUSS against attack_oracle at the tolerance of
  test_attacks_gpu.py.

Every output is pre-filled with NaN; the part a call may write is compared bitwise (a zero by value: -0 and +0 are
tied in every order statistic), and everything else must still be NaN."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import attack_oracle as AT                              # noqa: E402
import coord_oracle as CO                               # noqa: E402
from kernel_util import close, load_kernels, rand_net, synth, to_dev   # noqa: E402

NAN = float("nan")
RULES = ("clip", "trim", "wmsr")


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def same(got, want, tag):
    """Bitwise equality, a zero compared by value; no NaN may be expected (it could not be told from the pre-fill)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, tag
    assert not np.isnan(want).any(), f"{tag}: the reference is NaN"
    g, w = got.view(np.uint32).copy(), want.view(np.uint32).copy()
    g[got == 0] = 0
    w[want == 0] = 0
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, f"{tag}: {bad.size} of {got.size} differ, first at {bad[:4]}: got {got[bad[:4]]} want {want[bad[:4]]}"


def untouched(buf, tag):
    assert np.isnan(buf).all(), f"{tag}: wrote outside its range"


def valid_H(rule, n):
    return range(0, (n - 1) // 2 + 1) if rule == "trim" else range(0, n)


# ---------------------------------------------------------------------------------------------------------- clip_mean
CM_N = (7, 8, 9, 15, 16, 17, 24, 25, 64, 65, 129)
CM_P = (1, 2, 3, 4, 5, 7, 8, 255, 256, 257, 1024, 1025)
PMAX = max(CM_P)
SA, SO = 1028, 1029                                      # row strides: aligned (a multiple of 4) and odd
OB = 1032                                                # output slot per launch (a multiple of 4 floats)


def cm_columns(rs, n, H, P=PMAX):
    """n x P fp32: column kinds in a random order -- Gaussian rows of different scales, small-integer ties, every row
    equal to own, half the rows equal to own, and outlier columns with <= H entries of 1e8, +-1e30 or +-inf in
    non-own rows (Gaussian columns when H = 0)."""
    X = (rs.randn(n, P) * rs.uniform(0.1, 3.0, size=(n, 1))).astype(np.float32)
    kind = rs.permutation(np.arange(P) % 6)
    X[:, kind == 1] = rs.randint(-2, 3, size=(n, int((kind == 1).sum())))
    X[:, kind == 2] = X[0, kind == 2]
    half = (rs.rand(n, P) < 0.5) & (kind == 3)
    X = np.where(half, X[0], X)
    for c in np.flatnonzero(kind >= 4):
        if H == 0:
            continue
        k = int(rs.randint(1, H + 1)) if kind[c] == 4 else H
        rows = rs.choice(np.arange(1, n), size=k, replace=False)
        X[rows, c] = rs.choice([1e8, -1e8, 1e30, -1e30, np.inf, -np.inf], size=k)
    return X.astype(np.float32)


class ClipLayouts:
    """One n x PMAX input in two layouts: aligned (row stride SA at a 16-byte boundary) and offset (one float past it,
    row stride SO); every launch writes to its own NaN-filled output slot, aligned or one float past it."""

    def __init__(self, K, X, n_launch):
        n = X.shape[0]
        a = np.full(n * SA, NAN, np.float32)
        o = np.full(1 + n * SO, NAN, np.float32)
        for k in range(n):
            a[k * SA: k * SA + PMAX] = X[k]
            o[1 + k * SO: 1 + k * SO + PMAX] = X[k]
        self.a, self.o = to_dev(K, a, o)
        self.out = torch.full((n_launch, OB), NAN, device=K.dev)
        self.n = n

    def vals(self, layout, P):
        if layout == "aligned":
            return self.a.view(self.n, SA)[:, :P]
        return self.o[1:].view(self.n, SO)[:, :P]

    def run(self, K, slot, layout, P, H):
        vals = self.vals(layout, P)
        out = self.out[slot, :P] if layout == "aligned" else self.out[slot, 1:1 + P]
        K.ops.clip_mean(vals, H, out=out)
        w = CO.vec_width(H)
        vec = (P % w == 0 and vals.stride(0) % w == 0 and vals.data_ptr() % (4 * w) == 0 and out.data_ptr() % (4 * w) == 0)
        return w if vec else 1


def check_slot(buf, layout, P, want, tag):
    lo = 0 if layout == "aligned" else 1
    same(buf[lo:lo + P], want, tag)
    untouched(np.concatenate([buf[:lo], buf[lo + P:]]), tag)


@pytest.mark.parametrize("H", range(0, 8))
def test_clip_mean_bitwise_at_every_shape_and_path(K, H):
    rs = np.random.RandomState(6100 + H)
    n_vec = n_second = 0
    for n in sorted({H + 1} | {n for n in CM_N if n > H}):
        X = cm_columns(rs, n, H)
        L = ClipLayouts(K, X, 2 * len(CM_P))
        cases = []
        for i, P in enumerate(CM_P):
            for j, layout in enumerate(("aligned", "offset")):
                cases.append((2 * i + j, layout, P, L.run(K, 2 * i + j, layout, P, H)))
        got = L.out.cpu().numpy()
        srt = np.sort(X, axis=0)
        for slot, layout, P, vec in cases:
            want, second = CO.clip_mean(X[:, :P], H, vec, paths=True, srt=srt[:, :P])
            check_slot(got[slot], layout, P, want, f"H={H} n={n} P={P} {layout} vec={vec}")
            n_vec += vec > 1
            n_second += int(second.any())
        assert cases[-1][3] == 1                                    # the offset layout is always scalar
    assert n_vec >= 8 and (H == 0 or n_second >= 8), (n_vec, n_second)


@pytest.mark.parametrize("scale", CO.INT_SCALES, ids=list(CO.INT_SCALES))
def test_clip_mean_integer_columns_match_the_closed_form(K, scale):
    """Exact sums: one IEEE division per column, subnormal at 2^-140 (a flush-to-zero or approximate division fails)."""
    rs = np.random.RandomState(6200)
    s = CO.INT_SCALES[scale]
    for H in range(0, 8):
        for n in (H + 1, 9, 17, 65):
            if n <= H:
                continue
            ints, X = CO.int_columns(rs, n, 1024, s)
            want = CO.clip_closed(ints, H, s)
            if scale == "subnormal":
                assert ((want != 0) & (np.abs(want) < 2.0 ** -126)).sum() > 100
            L = ClipLayouts(K, np.pad(X, ((0, 0), (0, PMAX - 1024))), 2)
            for slot, layout in enumerate(("aligned", "offset")):
                vec = L.run(K, slot, layout, 1024, H)
                assert vec == (CO.vec_width(H) if layout == "aligned" else 1)
            got = L.out.cpu().numpy()
            for slot, layout in enumerate(("aligned", "offset")):
                check_slot(got[slot], layout, 1024, want, f"{scale} H={H} n={n} {layout}")


def test_clip_mean_c5_shape_every_H(K):
    """64 x 1 048 576 (the C5 microbenchmark), aligned: the vector kernel, with outlier columns in the first 8192."""
    n, P = 64, 1 << 20
    g = np.random.default_rng(6300)
    X = g.standard_normal((n, P), dtype=np.float32)
    X *= g.uniform(0.1, 3.0, size=(n, 1)).astype(np.float32)
    X[:, 1::9] = np.round(X[:, 1::9])                                  # ties
    X[:, 2::9] = X[0, 2::9]                                            # equal to own
    dX = to_dev(K, X)[0]
    srt = np.sort(X, axis=0)
    out = torch.full((P + 8,), NAN, device=K.dev)
    for H in range(0, 8):
        Xh = X
        if H:
            Xh = X.copy()
            cols = np.arange(0, 8192, 3)
            for i in range(H):
                Xh[g.integers(1, n, size=cols.size), cols] = g.choice(np.float32([1e8, -1e30, np.inf, -np.inf]), size=cols.size)
            dX[:, :8192] = to_dev(K, np.ascontiguousarray(Xh[:, :8192]))[0]
        out.fill_(NAN)
        K.ops.clip_mean(dX, H, out=out[:P])
        got = out.cpu().numpy()
        s = srt if H == 0 else np.concatenate([np.sort(Xh[:, :8192], axis=0), srt[:, 8192:]], 1)
        want, second = CO.clip_mean(Xh, H, CO.vec_width(H), paths=True, srt=s)
        same(got[:P], want, f"C5 H={H}")
        untouched(got[P:], f"C5 H={H}")
        assert H == 0 or second[:8192].sum() > 1000
        if H:
            dX[:, :8192] = to_dev(K, np.ascontiguousarray(X[:, :8192]))[0]


# ---------------------------------------------------------------------------------------------------------- consensus
NR, NBYZ = 24, 4                                         # message rows; the last NBYZ carry +-inf / +-1e30
MS, MOFF = 1403, 3                                       # odd message stride, odd offset
DS, DOFF = 1411, 5                                       # output slot per job and offset within it
NH = (1, 255, 256, 257, 1400)


def message_rows(rs, P):
    """NR rows of P floats: Gaussian coordinates, small-integer ties and coordinates equal in every row; the Byzantine
    rows hold +-inf or +-1e30 at about a third of their coordinates."""
    X = (rs.randn(NR, P) * rs.uniform(0.1, 3.0, size=(NR, 1))).astype(np.float32)
    kind = rs.randint(0, 3, size=P)
    X[:, kind == 1] = rs.randint(-2, 3, size=(NR, int((kind == 1).sum())))
    X[:, kind == 2] = X[0, kind == 2]
    bad = rs.rand(NBYZ, P) < 0.35
    X[NR - NBYZ:] = np.where(bad, rs.choice(np.float32([np.inf, -np.inf, 1e30, -1e30]), size=(NBYZ, P)), X[NR - NBYZ:])
    return X.astype(np.float32)


def in_nodes(rs, n_in, H):
    """own first (an honest row), repeats allowed, at most H slots on Byzantine rows (H of them about half the time)."""
    honest = NR - NBYZ
    nodes = [int(rs.randint(0, honest))] + [int(x) for x in rs.randint(0, honest, size=n_in - 1)]
    if n_in >= 3:
        nodes[int(rs.randint(1, n_in))] = nodes[0]
    n_byz = H if rs.rand() < 0.5 else int(rs.randint(0, H + 1))
    for slot in rs.choice(np.arange(1, n_in), size=min(n_byz, n_in - 1), replace=False):
        nodes[int(slot)] = int(rs.randint(NR - NBYZ, NR))
    return nodes


def test_consensus_hidden_every_rule_n_in_and_H(K):
    rs = np.random.RandomState(6400)
    X = message_rows(rs, max(NH))
    flat = np.full(MOFF + NR * MS, NAN, np.float32)
    for r in range(NR):
        flat[MOFF + r * MS: MOFF + r * MS + X.shape[1]] = X[r]
    msgs = to_dev(K, flat)[0][MOFF:]
    cases = [(rule, n_in, H, nh) for rule in RULES for n_in in range(1, 17) for H in valid_H(rule, n_in) for nh in NH]
    order = rs.permutation(len(cases))                       # every launch mixes rules, n_in and n_hidden
    cases = [cases[i] + (in_nodes(rs, cases[i][1], cases[i][2]),) for i in order]
    dst = torch.full((len(cases), DS), NAN, device=K.dev)
    for b in range(0, len(cases), 32):
        K.ops.consensus_hidden([K.ops.consensus_job(dst[j, DOFF:], msgs, MS, nh, nodes, H, rule)
                                for j, (rule, n_in, H, nh, nodes) in enumerate(cases[b:b + 32], b)])
    got = dst.cpu().numpy()
    for j, (rule, n_in, H, nh, nodes) in enumerate(cases):
        tag = f"{rule} n_in={n_in} H={H} n_hidden={nh} nodes={nodes}"
        same(got[j, DOFF:DOFF + nh], CO.resilient_mean_small(X[nodes, :nh], H, rule), tag)
        assert np.isfinite(got[j, DOFF:DOFF + nh]).all(), tag
        untouched(np.concatenate([got[j, :DOFF], got[j, DOFF + nh:]]), tag)
    assert len(cases) > 1700


# ---------------------------------------------------------------------------------------------------------- team
N_HEADS = 40                                             # head messages; the last 8 predict +-inf or +-1e30


def head_stack(K, rs, din, b3):
    """Packed networks of din inputs with W3 = 0 and b3 = b3[m]: every estimate of head m is exactly b3[m]."""
    rows = []
    for v in b3:
        w = rand_net(rs, din, 1)
        w[4] = np.zeros_like(w[4])
        w[5] = np.full_like(w[5], v)
        rows.append(K.nets.pack(w))
    return to_dev(K, np.stack(rows))[0]


def head_values(rs):
    v = (rs.randn(N_HEADS) * 2).astype(np.float32)
    v[:12] = rs.randint(-2, 3, size=12)                     # ties
    v[12:14] = [2.0 ** -140, -3 * 2.0 ** -140]              # subnormal
    v[N_HEADS - 8:] = [np.inf, -np.inf, 1e30, -1e30, np.inf, -np.inf, 1e30, -1e30]
    return v.astype(np.float32)


def head_nodes(rs, n_in, H):
    nodes = [int(x) for x in rs.randint(0, N_HEADS - 8, size=n_in)]
    if n_in >= 3:
        nodes[int(rs.randint(1, n_in))] = nodes[0]
    n_byz = min(H, n_in - 1) if rs.rand() < 0.5 else int(rs.randint(0, min(H, n_in - 1) + 1))
    for slot in rs.choice(np.arange(1, n_in), size=n_byz, replace=False):
        nodes[int(slot)] = int(rs.randint(N_HEADS - 8, N_HEADS))
    return nodes


@pytest.mark.parametrize("NA", [5, 16])
def test_team_agg_out_exact_on_every_row(K, NA):
    rs = np.random.RandomState(6500 + NA)
    T = 1200
    s, ns, a, r = synth(rs, T, NA, 5 if NA == 5 else 10)
    dsa, dns, dr = to_dev(K, np.concatenate([s, a], -1).reshape(T, -1), ns.reshape(T, -1), r[:, :, 0])
    b3 = head_values(rs)
    dins = {K.L.IN_S: 2 * NA, K.L.IN_SA: 3 * NA, K.L.IN_NS: 2 * NA}
    stacks = {d: head_stack(K, rs, d, b3) for d in set(dins.values())}
    own = {d: to_dev(K, K.nets.pack(rand_net(rs, d, 1)))[0] for d in set(dins.values())}
    cases = []
    for rule in RULES:
        for n_in in range(1, 17):
            Hs = list(valid_H(rule, n_in))
            for H in sorted({Hs[-1], Hs[int(rs.randint(0, len(Hs)))]}):
                kind = (K.L.IN_S, K.L.IN_SA, K.L.IN_NS)[len(cases) % 3]
                cases.append((rule, n_in, H, kind, head_nodes(rs, n_in, H)))
    perm = rs.permutation(len(cases))
    cases = [cases[i] for i in perm]
    tidx = to_dev(K, rs.choice(400, size=57, replace=False).astype(np.int32))[0]
    for rows_kw in (dict(row_begin=37, n_rows=100), dict(row_begin=5, n_rows=1001),
                    dict(time_idx=tidx, n_envs=3, n_rows=171)):
        rows = K.ops.make_rows(dsa, dns, dr, NA, **rows_kw)
        if "time_idx" in rows_kw:
            t = tidx.cpu().numpy().astype(np.int64)
            live = (t[:, None] * 3 + np.arange(3)).reshape(-1)
        else:
            live = rows_kw["row_begin"] + np.arange(rows_kw["n_rows"])
        agg = torch.full((len(cases), T), NAN, device=K.dev)
        for b in range(0, len(cases), 32):
            jobs = []
            for j, (rule, n_in, H, kind, nodes) in enumerate(cases[b:b + 32], b):
                d = dins[kind]
                jobs.append(K.ops.team_job(own[d], kind, stacks[d], stacks[d].shape[1], nodes, H, agg_out=agg[j],
                                           rule=rule))
            K.ops.team(rows, jobs)
        got = agg.cpu().numpy()
        dead = np.ones(T, bool)
        dead[live] = False
        for j, (rule, n_in, H, kind, nodes) in enumerate(cases):
            tag = f"NA={NA} {rows_kw.get('n_rows')} rows {rule} n_in={n_in} H={H} kind={kind} nodes={nodes}"
            want = CO.resilient_mean_small(b3[nodes][:, None], H, rule)
            assert np.isfinite(want).all(), tag
            same(got[j, live], np.repeat(want, live.size), tag)
            untouched(got[j, dead], tag)


# ---------------------------------------------------------------------------------------------------------- attack
AP = (1, 255, 256, 257, 1421)
AS, AOFF = 1433, 3                                      # odd message stride and offset
ADS, ADOFF = 1433, 1                                    # output slot per job and offset within it


def attack_stack(K, X):
    flat = np.full(AOFF + X.shape[0] * AS, NAN, np.float32)
    for r in range(X.shape[0]):
        flat[AOFF + r * AS: AOFF + r * AS + X.shape[1]] = X[r]
    return to_dev(K, flat)[0][AOFF:]


def run_attacks(K, msgs, specs):
    """specs: (kind, param, n, honest, counter kwargs); 32 jobs per launch; returns the output slots."""
    dst = torch.full((len(specs), ADS), NAN, device=K.dev)
    for b in range(0, len(specs), 32):
        K.ops.attack([K.ops.attack_job(dst[j, ADOFF:], msgs, AS, n, honest, kind, param, **ctr)
                      for j, (kind, param, n, honest, ctr) in enumerate(specs[b:b + 32], b)])
    return dst.cpu().numpy()


def test_alie_and_ipm_bitwise(K):
    rs = np.random.RandomState(6600)
    X = (rs.randn(20, max(AP)) * rs.uniform(0.1, 3.0, size=(20, 1))).astype(np.float32)
    X[:, ::5] = rs.randint(-2, 3, size=(20, X[:, ::5].shape[1]))
    X[:, 1::7] = X[0, 1::7]
    msgs = attack_stack(K, X)
    specs = []
    for kind in ("alie", "ipm"):
        for n_h in range(1, 17):
            for i, n in enumerate(AP):
                honest = [int(x) for x in rs.randint(0, 20, size=n_h)]
                if n_h >= 3:
                    honest[-1] = honest[0]
                param = float([1.5, -0.7, 3.0, 0.0, 0.25, 1.0, -2.0, 0.5, 2.75, -1.3][(n_h + i) % 10])
                ctr = dict(seed=99 + n_h, attacker=255 if i % 2 else n_h, receiver=255 if i % 3 == 0 else 7)
                specs.append((kind, param, n, honest, ctr))
    specs = [specs[i] for i in rs.permutation(len(specs))]
    got = run_attacks(K, msgs, specs)
    for j, (kind, param, n, honest, ctr) in enumerate(specs):
        tag = f"{kind} {param} n={n} honest={honest}"
        same(got[j, ADOFF:ADOFF + n], CO.attack(X[honest, :n], kind, param), tag)
        untouched(np.concatenate([got[j, :ADOFF], got[j, ADOFF + n:]]), tag)


@pytest.mark.parametrize("scale", CO.ATTACK_SCALES, ids=list(CO.ATTACK_SCALES))
def test_alie_and_ipm_on_symmetric_rows_match_the_closed_form(K, scale):
    rs = np.random.RandomState(6700)
    s = CO.ATTACK_SCALES[scale]
    specs, want = [], []
    blocks, r0 = [], 0
    for n_h in (2, 4, 6, 16):
        Xb, c, a = CO.symmetric_rows(rs, n_h, max(AP), s)
        blocks.append(Xb)
        for z in (0.0, 1.0, -1.0, 2.0, -2.0, 0.5, 1.5):
            specs.append(("alie", z, max(AP), list(range(r0, r0 + n_h)), {}))
            want.append(CO.alie_closed(c, a, z, s))
            specs.append(("ipm", z, max(AP), list(range(r0, r0 + n_h))[::-1], {}))
            want.append(CO.ipm_closed(c, z, s))
        r0 += n_h
    X = np.concatenate(blocks)
    got = run_attacks(K, attack_stack(K, X), specs)
    for j, ((kind, z, n, honest, _), w) in enumerate(zip(specs, want)):
        same(got[j, ADOFF:ADOFF + n], w, f"{scale} {kind} {z} n_honest={len(honest)}")
        same(got[j, ADOFF:ADOFF + n], CO.attack(X[honest, :n], kind, z), f"{scale} {kind} {z} restatement")


def test_gauss_against_the_oracle(K):
    rs = np.random.RandomState(6800)
    X = (rs.randn(20, max(AP)) * rs.uniform(0.1, 3.0, size=(20, 1))).astype(np.float32)
    msgs = attack_stack(K, X)
    specs = []
    for n_h in range(1, 17):
        for i, n in enumerate(AP[n_h % 2::2]):
            honest = [int(x) for x in rs.randint(0, 20, size=n_h)]
            ctr = dict(seed=(5 << 32) + n_h, attacker=255 if i == 0 else n_h, receiver=255 if n_h % 2 else 3,
                       round=1000 + i, epoch=n_h % 4)
            specs.append(("gauss", float([0.3, 0.0, 2.0][(n_h + i) % 3]), n, honest, ctr))
    got = run_attacks(K, msgs, specs)
    for j, (kind, param, n, honest, ctr) in enumerate(specs):
        vals = X[honest, :n].astype(np.float64)
        xi = AT.gauss_xi(n, ctr["seed"], ctr["attacker"], ctr["receiver"], ctr["round"], ctr["epoch"])
        tag = f"gauss {param} n={n} honest={honest}"
        close(got[j, ADOFF:ADOFF + n], AT.craft(vals, "gauss", param, xi), rtol=0,
              atol=4e-6 * max(np.abs(vals).max(), 1.0) * (1 + abs(param)), err_msg=tag)
        untouched(np.concatenate([got[j, :ADOFF], got[j, ADOFF + n:]]), tag)
