"""The whole-message kernels (rcmarl_vector_aggregate, rcmarl_dnc_aggregate, rcmarl_nnm_mix, rcmarl_bucket_mix,
rcmarl_adaptive_attack, rcmarl_tailored_attack, rcmarl_pipeline_attack, rcmarl_dissensus_attack, rcmarl_mimic_attack) at
the edges of their ABI:

- a parameter-count sweep, P in edge_inputs.SWEEP_P (1, 2, 3, below / at / past a warp and a block, and 1421), every
  launch holding P = 1 and P = 1421 jobs (its dynamic shared memory sized by the largest), against the fp64 oracles
  with the tolerances and margin rules of each entry point's own test file;
- exact answers on integer-valued messages from tests/edge_inputs.py: identical messages, two clusters, rows on a
  line, repeated in-nodes, one parameter, squared distances that overflow to +inf or underflow to 0 in fp32 --
  selections, weights and outputs compared bitwise with the closed forms, with no margin escape;
- the per-agent API (RPBCAC_agent._resilient_aggregation) on (n, 1) and (n, 2, 3) tensors.

Every message stack starts at an odd float offset with a row stride wider than P (NaN in between), every output at
another odd offset; outputs and weights are pre-filled with NaN and everything past what a job may write must stay
NaN."""
import collections

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                     # noqa: E402
import bucket_oracle as BO                              # noqa: E402
import dissensus_mimic_oracle as DM                     # noqa: E402
import dnc_oracle as DO                                 # noqa: E402
import edge_inputs as E                                 # noqa: E402
import nnm_oracle as NO                                 # noqa: E402
import pipeline_attack_oracle as PA                     # noqa: E402
import tailored_attack_oracle as TA                     # noqa: E402
import test_pipeline_attack_gpu as PG                   # noqa: E402  (the pipeline checker)
import test_tailored_attacks_gpu as TG                  # noqa: E402  (the tailored checker)
import vector_oracle as VO                              # noqa: E402
from kernel_util import close, load_kernels             # noqa: E402

f64 = np.float64
NAN = float("nan")
S = 1441                                                # row stride: odd, wider than every P
IN_OFF, OUT_OFF, W_OFF = 3, 5, 1
PMAX = max(E.SWEEP_P)
MARGIN, G_RTOL, PICK_GAP = 1e-4, 5e-5, 1e-4


@pytest.fixture(scope="module")
def K():
    return load_kernels()


# ---------------------------------------------------------------------------------------------------------- layout
class Stack:
    """Row blocks [n_i, P_i] stored one after another at IN_OFF + r * S of a NaN-filled device buffer."""

    def __init__(self, K, blocks):
        self.rows = []
        r = 0
        for b in blocks:
            self.rows.append(list(range(r, r + b.shape[0])))
            r += b.shape[0]
        flat = np.full(IN_OFF + r * S, np.nan, np.float32)
        for b, ids in zip(blocks, self.rows):
            for x, i in zip(b, ids):
                flat[IN_OFF + i * S: IN_OFF + i * S + x.shape[0]] = x
        self.dev = torch.as_tensor(flat).to(K.dev)
        self.msgs = self.dev[IN_OFF:]


def outputs(K, n_jobs, n_rows=1):
    return torch.full((n_jobs, OUT_OFF + n_rows * S), NAN, device=K.dev)


def written(buf, n_rows, P, tag):
    """The [n_rows, P] rows a job wrote at OUT_OFF + r * S of its buffer row; everything else must still be NaN."""
    buf = buf.copy()
    got = np.stack([buf[OUT_OFF + r * S: OUT_OFF + r * S + P].copy() for r in range(n_rows)])
    for r in range(n_rows):
        buf[OUT_OFF + r * S: OUT_OFF + r * S + P] = np.nan
    assert np.isnan(buf).all(), f"{tag}: wrote outside its rows"
    return got


def wslice(buf, n, tag):
    assert np.isnan(buf[:W_OFF]).all() and np.isnan(buf[W_OFF + n:]).all(), f"{tag}: wrote past its weights"
    return buf[W_OFF:W_OFF + n]


def _gauss(rs, n_rows=24, P=PMAX):
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def _sweep_jobs(rs, n_ins, n_rows=24):
    """(P, n_in, nodes) for every P of the sweep and each n_in of n_ins (a tuple entry cycles over the P), some with a
    repeated in-node."""
    out = []
    for i, P in enumerate(E.SWEEP_P):
        for j, n_in in enumerate(n_ins):
            n_in = n_in[i % len(n_in)] if isinstance(n_in, tuple) else n_in
            nodes = [int(x) for x in rs.choice(n_rows, size=n_in, replace=False)]
            if n_in >= 3 and (i + j) % 3 == 0:
                nodes[-1] = nodes[1]
            out.append((P, n_in, nodes))
    return out


# ---------------------------------------------------------------------------------------------------------- a) sweep
@pytest.mark.parametrize("rules", [("krum", "mkrum"), ("scclip", "gmed")])
def test_vector_aggregate_parameter_sweep(K, rules):
    rs = np.random.RandomState(8100)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = [(rules[(i // 2) % 2], P, n_in, nodes) for i, (P, n_in, nodes) in
             enumerate(_sweep_jobs(rs, (16, 3) if rules[0] == "krum" else (16, 1)))]
    dst, wout = outputs(K, len(cases)), torch.full((len(cases), 24), NAN, device=K.dev)
    jobs = []
    for j, (rule, P, n_in, nodes) in enumerate(cases):
        H = {"krum": n_in - 3, "mkrum": (n_in - 3) // 2, "scclip": n_in // 3, "gmed": 0}[rule]
        jobs.append(K.ops.vector_job(dst[j, OUT_OFF:], st.msgs, S, P, nodes, H, rule, weights_out=wout[j, W_OFF:]))
        cases[j] = (rule, P, n_in, nodes, H)
    K.ops.vector_aggregate(jobs)
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (rule, P, n_in, nodes, H) in enumerate(cases):
        tag = f"{rule} P={P} n_in={n_in} H={H} nodes={nodes}"
        out, w = written(got[j], 1, P, tag)[0], wslice(gw[j], n_in, tag)
        Xj = X[nodes, :P].astype(f64)
        want, ww = VO.aggregate(Xj, H, rule)
        if rule in ("krum", "mkrum"):
            m = 1 if rule == "krum" else n_in - H
            s = np.sort(VO.krum_scores(Xj, H))
            mg = np.inf if m == n_in else (s[m] - s[m - 1]) / max(s[m], 1e-300)
            if mg > MARGIN or mg == 0:
                np.testing.assert_array_equal(w > 0, ww > 0, err_msg=tag)
            else:
                want = Xj[w > 0].mean(0)
            close(out, want, rtol=0, atol=4e-6 * max(np.abs(Xj).max(), 1.0), err_msg=tag)
        else:
            if not (rule == "gmed" and len(set(nodes)) < n_in):
                close(w, ww, rtol=0, atol=1e-5 if rule == "scclip" else 1e-4 * np.abs(ww).max(), err_msg=tag)
            close(out, want, rtol=0, atol=2e-5 * max(np.abs(Xj).max(), 1.0), err_msg=tag)


def test_dnc_parameter_sweep(K):
    rs = np.random.RandomState(8200)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = _sweep_jobs(rs, (16, (1, 2), 9))
    dst, wout = outputs(K, len(cases)), torch.full((len(cases), 24), NAN, device=K.dev)
    Hs = [(n_in - 1) if i % 3 == 0 else n_in // 2 for i, (_, n_in, _) in enumerate(cases)]
    K.ops.dnc_aggregate([K.ops.vector_job(dst[j, OUT_OFF:], st.msgs, S, P, nodes, Hs[j], K.L.SPECTRAL_DNC,
                                          weights_out=wout[j, W_OFF:]) for j, (P, n_in, nodes) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    n_exact = 0
    for j, (P, n_in, nodes) in enumerate(cases):
        H = Hs[j]
        tag = f"dnc P={P} n_in={n_in} H={H} nodes={nodes}"
        out, w = written(got[j], 1, P, tag)[0], wslice(gw[j], n_in, tag)
        Xj = X[nodes, :P].astype(f64)
        want, ww = DO.aggregate(Xj, H)
        assert (w > 0).sum() == n_in - H, tag
        eig, gap = DO.margins(Xj, H)
        if eig >= 1e-3 and gap >= 1e-6:
            n_exact += 1
            np.testing.assert_array_equal(w > 0, ww > 0, err_msg=tag)
        else:
            want = Xj[w > 0].mean(0)
        close(out, want, rtol=0, atol=4e-6 * max(np.abs(Xj).max(), 1.0), err_msg=tag)
    assert n_exact >= 0.8 * len(cases), n_exact


def test_nnm_parameter_sweep(K):
    rs = np.random.RandomState(8300)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = _sweep_jobs(rs, (16, 1, 5))
    dst, wout = outputs(K, len(cases), 16), torch.full((len(cases), 260), NAN, device=K.dev)
    Hs = [(i * 7) % n_in for i, (_, n_in, _) in enumerate(cases)]
    K.ops.nnm_mix([K.ops.vector_job(dst[j, OUT_OFF:], st.msgs, S, P, nodes, Hs[j], K.L.MIX_NNM,
                                    weights_out=wout[j, W_OFF:]) for j, (P, n_in, nodes) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (P, n_in, nodes) in enumerate(cases):
        H = Hs[j]
        tag = f"nnm P={P} n_in={n_in} H={H} nodes={nodes}"
        mixed, M = written(got[j], n_in, P, tag), wslice(gw[j], n_in * n_in, tag).reshape(n_in, n_in)
        Xj = X[nodes, :P].astype(f64)
        sel = None if NO.clear(Xj, H) else [list(np.flatnonzero(r > 0)) for r in M]
        want, WM = NO.mix(Xj, H, sel)
        np.testing.assert_array_equal(M > 0, WM > 0, err_msg=tag)
        close(mixed, want, rtol=0, atol=4e-6 * max(np.abs(Xj).max(), 1.0), err_msg=tag)


def test_bucket_parameter_sweep(K):
    rs = np.random.RandomState(8400)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = _sweep_jobs(rs, (16, 1, 4))
    ss = [1 + i % 4 for i in range(len(cases))]
    words = [dict(seed=2 ** 33 + i, receiver=i % 7, net=i % 2, round=3 * i, epoch=i % 5) for i in range(len(cases))]
    dst, wout = outputs(K, len(cases), 16), torch.full((len(cases), 260), NAN, device=K.dev)
    K.ops.bucket_mix([K.ops.bucket_job(dst[j, OUT_OFF:], st.msgs, S, P, nodes, ss[j], weights_out=wout[j, W_OFF:],
                                       **words[j]) for j, (P, n_in, nodes) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (P, n_in, nodes) in enumerate(cases):
        n_out = BO.n_out(n_in, ss[j])
        tag = f"bucket P={P} n_in={n_in} s={ss[j]} nodes={nodes}"
        rows, M = written(got[j], n_out, P, tag), wslice(gw[j], n_out * n_in, tag).reshape(n_out, n_in)
        Xj = X[nodes, :P]
        w = words[j]
        want, WM = BO.bucket_mix(Xj.astype(f64), ss[j], w["seed"], w["receiver"], w["net"], w["round"], w["epoch"])
        np.testing.assert_array_equal(M, WM.astype(np.float32), err_msg=tag)
        np.testing.assert_array_equal(rows[0], Xj[0], err_msg=tag)
        close(rows, want, rtol=0, atol=4e-6 * max(np.abs(Xj).max(), 1.0), err_msg=tag)


def test_adaptive_attack_parameter_sweep(K):
    rs = np.random.RandomState(8500)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = [(AA.ATTACKS[i % 6], P, nodes) for i, (P, _, nodes) in enumerate(_sweep_jobs(rs, (16, 1, 2)))]
    dst, gam = outputs(K, len(cases)), torch.full((len(cases), 3), NAN, device=K.dev)
    K.ops.adaptive_attack([K.ops.adaptive_attack_job(dst[j, OUT_OFF:], st.msgs, S, P, h, a, 1.0,
                                                     gamma_out=gam[j, 1:2]) for j, (a, P, h) in enumerate(cases)])
    got, gg = dst.cpu().numpy(), gam.cpu().numpy()
    for j, (attack, P, honest) in enumerate(cases):
        tag = f"{attack} P={P} honest={honest}"
        msg = written(got[j], 1, P, tag)[0]
        assert np.isnan(gg[j, 0]) and np.isnan(gg[j, 2]), tag
        V = X[honest, :P].astype(f64)
        want, g = AA.craft(V, attack, 1.0)
        if len(set(honest)) == 1:
            assert gg[j, 1] == 0 and np.array_equal(msg, X[honest[0], :P]), tag
            continue
        close(gg[j, 1], g, rtol=G_RTOL, atol=0, err_msg=tag)
        d = AA.gamma_of(V, attack)[1]
        close(msg, want, rtol=0, atol=1e-5 * max(np.abs(V).max(), 1.0) + G_RTOL * g * np.abs(d).max(), err_msg=tag)


def _attack_cases(rs, rules, n_rows=24):
    """(attack dev, rule, H, slots, honest, P) per P of the sweep: n_in 2 and 16 (krum: 3 and 16)."""
    out = []
    for i, P in enumerate(E.SWEEP_P):
        for j, n_in in enumerate((16, 2)):
            rule = rules[(2 * i + j) % len(rules)]
            n_in = max(n_in, 3) if rule in ("krum", "mkrum") else n_in
            rows = [int(x) for x in rs.choice(n_rows, size=n_in, replace=False)]
            n_cr = 1 + (i + j) % 3 if n_in > 4 else 1
            slots = rows[:n_in - n_cr] + [-1] * n_cr
            honest = list(range(n_in - n_cr - (n_in > 4)))
            H = min(1 + i % 2, TG._max_h(rule, n_in) if rule != "dnc" else n_in - 1)
            out.append((("uv", "std", "sgn")[(i + j) % 3], rule, H, slots, honest, P))
    return out


def test_tailored_attack_parameter_sweep(K):
    rs = np.random.RandomState(8600)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = [("tailored_" + a, r, H, s, h, P) for a, r, H, s, h, P in
             _attack_cases(rs, ("clip", "krum", "trim", "gmed", "mkrum", "scclip", "wmsr"))]
    dst, gam = outputs(K, len(cases)), torch.full((len(cases), 2), NAN, device=K.dev)
    K.ops.tailored_attack([K.ops.tailored_attack_job(dst[j, OUT_OFF:], st.msgs, S, P, s, h, r, H, a, 2.0,
                                                     gamma_out=gam[j, :1]) for j, (a, r, H, s, h, P) in enumerate(cases)])
    got, gg = dst.cpu().numpy(), gam.cpu().numpy()
    stats = collections.Counter()
    for j, case in enumerate(cases):
        msg = written(got[j], 1, case[-1], str(case))[0]
        TG._check_job(np.concatenate([msg, [NAN]]), gg[j], X, case, 2.0, stats)


def test_pipeline_attack_parameter_sweep(K):
    rs = np.random.RandomState(8700)
    X = _gauss(rs)
    st = Stack(K, [X])
    mixings = (None, "nnm", ("bucket", 2), ("bucket", 3))
    cases = []
    for c, (a, r, H, s, h, P) in enumerate(_attack_cases(rs, ("dnc", "clip", "mkrum", "dnc", "gmed", "trim"))):
        mixing = mixings[c % 4] if len(s) > 2 else None
        n_rows = PA.n_rows(len(s), mixing)
        if r in ("krum", "mkrum") and n_rows < 3:
            mixing, n_rows = None, len(s)
        H = min(H, n_rows - 1 if r == "dnc" else TG._max_h(r, n_rows))
        cases.append(("pipeline_" + a, r, H, s, h, P, mixing))
    dst, gam = outputs(K, len(cases)), torch.full((len(cases), 2), NAN, device=K.dev)
    mod = outputs(K, len(cases))
    words = dict(PG.WORDS)
    words["round"] = words.pop("round_")
    K.ops.pipeline_attack([K.ops.pipeline_attack_job(dst[j, OUT_OFF:], st.msgs, S, P, s, h, r, H, a, 2.0, mixing=m,
                                                     n_perms=3, gamma_out=gam[j, :1], model_out=mod[j, OUT_OFF:],
                                                     **words) for j, (a, r, H, s, h, P, m) in enumerate(cases)])
    got, gg, mo = dst.cpu().numpy(), gam.cpu().numpy(), mod.cpu().numpy()
    stats = collections.Counter()
    for j, case in enumerate(cases):
        P = case[5]
        msg = written(got[j], 1, P, str(case))[0]
        assert np.isnan(gg[j, 1]), case
        assert np.isfinite(written(mo[j], 1, P, str(case))).all(), case
        PG._check(np.concatenate([msg, [NAN]]), gg[j, 0], X, case, 2.0, stats)


def test_dissensus_and_mimic_parameter_sweep(K):
    rs = np.random.RandomState(8800)
    X = _gauss(rs)
    st = Stack(K, [X])
    cases = [(P, nodes) for P, _, nodes in _sweep_jobs(rs, (16, 1, 2))]
    dst = outputs(K, len(cases))
    spec = [(1 + j % 4, (0.5, 1.0, 2.5)[j % 3]) for j in range(len(cases))]
    K.ops.dissensus_attack([K.ops.dissensus_attack_job(dst[j, OUT_OFF:], st.msgs, S, P, h[0], h, *spec[j])
                            for j, (P, h) in enumerate(cases)])
    got = dst.cpu().numpy()
    for j, (P, h) in enumerate(cases):
        V = X[h, :P].astype(f64)
        n_byz, eps = spec[j]
        close(written(got[j], 1, P, f"dissensus P={P}")[0], DM.dissensus(V[0], V, n_byz, eps), rtol=0,
              atol=1e-6 * (1 + eps / n_byz * len(h)) * np.abs(V).max(), err_msg=f"dissensus P={P} {h}")
    # mimic: Init (update 0) then Init and a step (update 1), from z = 0
    for update in (0, 1):
        dst = outputs(K, len(cases))
        zb = torch.full((len(cases), OUT_OFF + S), NAN, device=K.dev)
        for j, (P, _) in enumerate(cases):
            zb[j, OUT_OFF:OUT_OFF + P] = 0
        tgt = torch.full((len(cases), 3), -7, dtype=torch.int32, device=K.dev)
        cands = [list(range(len(h))) if j % 2 else list(range(1, len(h))) or [0] for j, (_, h) in enumerate(cases)]
        K.ops.mimic_attack([K.ops.mimic_attack_job(dst[j, OUT_OFF:], st.msgs, S, P, h, cands[j], zb[j, OUT_OFF:],
                                                   update, target_out=tgt[j, 1:2]) for j, (P, h) in enumerate(cases)])
        got, zg, tg = dst.cpu().numpy(), zb.cpu().numpy(), tgt.cpu().numpy()
        for j, (P, h) in enumerate(cases):
            tag = f"mimic update={update} P={P} honest={h}"
            V = X[h, :P].astype(f64)
            zk = written(zg[j], 1, P, tag)[0]
            k0 = None
            if DM.init_margin(V) <= PICK_GAP:                # a near tie of e_k: follow the kernel's Init pick
                e = DM.init_scores(V)
                tied = [k for k in range(len(h)) if e[k] >= e.max() * (1 - PICK_GAP)]
                k0 = max(tied, key=lambda k: float(DM.mimic(V, cands[j], np.zeros(P), update, k0=k)[1] @ zk))
            k, z, t = DM.mimic(V, cands[j], np.zeros(P), update, k0=k0)
            assert tg[j, 0] == -7 and tg[j, 2] == -7, tag
            kg = int(tg[j, 1])
            assert kg in cands[j], tag
            np.testing.assert_array_equal(written(got[j], 1, P, tag)[0], X[h[kg], :P], err_msg=tag)
            close(zk, z, rtol=0, atol=1e-4, err_msg=tag)
            if DM.pick_margin(V, t) > PICK_GAP:
                assert np.array_equal(V[kg], V[k]), f"{tag}: copied {kg}, oracle {k}"


# ---------------------------------------------------------------------------------------------------------- b, c) exact
EDGE = E.edge_cases()
SCCLIP = [c for c in EDGE if c.P == 1 and not c.name.startswith("two") or c.name.split("_")[0] in
          ("identical", "overflow", "underflow")]


def _vector_edge_launch(K, cases, rule, fn):
    st = Stack(K, [c.X for c in cases])
    dst, wout = outputs(K, len(cases)), torch.full((len(cases), 24), NAN, device=K.dev)
    fam = K.ops.dnc_aggregate if rule == "dnc" else K.ops.vector_aggregate
    fam([K.ops.vector_job(dst[j, OUT_OFF:], st.msgs, S, c.P, st.rows[j], c.H,
                          K.L.SPECTRAL_DNC if rule == "dnc" else rule, weights_out=wout[j, W_OFF:])
         for j, c in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, c in enumerate(cases):
        tag = f"{rule} {c}"
        out, w = written(got[j], 1, c.P, tag)[0], wslice(gw[j], c.n, tag)
        ww, want = fn(c)
        np.testing.assert_array_equal(w, ww, err_msg=tag)
        np.testing.assert_array_equal(out, want, err_msg=tag)


@pytest.mark.parametrize("rule", ["krum", "mkrum"])
def test_krum_exact_answers(K, rule):
    """Every edge case, P = 1 and P = 1421 in one launch: selections by the tie rules, outputs bitwise."""
    _vector_edge_launch(K, EDGE, rule, lambda c: E.krum(c, rule))


def test_scclip_exact_answers(K):
    """P = 1 with distance ratios that are powers of two; identical rows (tau = 0, every c_k = 1, out = x_0); +inf
    distances (every c_k = 0, out = x_0); underflowing distances (d_k = 0 = tau, every c_k = 1)."""
    _vector_edge_launch(K, SCCLIP, "scclip", E.scclip)


def test_dnc_exact_answers(K):
    """Rows on a line (P = 1, collinear, two clusters, 2^64 and 2^-84 scales) and identical rows (G = 0, no rotation,
    equal scores: the H highest indices go) -- and every H on identical rows."""
    cases = [c for c in EDGE if c.t is not None]
    cases += [E.identical(P, H=H) for P in E.EDGE_P for H in (0, 1, 4, 6)]
    _vector_edge_launch(K, cases, "dnc", E.dnc)


def test_gmed_exact_answers(K):
    """+inf distances: only the median row is finite, out = that row, w = e_k; identical and underflowing rows: every
    beta_k equal (identical: out = x bitwise); collinear rows: on the line, as the fp64 Weiszfeld restatement."""
    cases = [E.scaled(P, E.OVER, "overflow") for P in E.EDGE_P] + [E.identical(P) for P in E.EDGE_P]
    cases += [E.scaled(P, E.UNDER, "underflow") for P in E.EDGE_P] + [E.collinear()]
    st = Stack(K, [c.X for c in cases])
    dst, wout = outputs(K, len(cases)), torch.full((len(cases), 24), NAN, device=K.dev)
    K.ops.vector_aggregate([K.ops.vector_job(dst[j, OUT_OFF:], st.msgs, S, c.P, st.rows[j], c.H, "gmed",
                                             weights_out=wout[j, W_OFF:]) for j, c in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, c in enumerate(cases):
        tag = f"gmed {c}"
        out, w = written(got[j], 1, c.P, tag)[0], wslice(gw[j], c.n, tag)
        kind = c.name.split("_")[0]
        if kind == "overflow":
            ww, want = E.gmed_overflow(c)
            np.testing.assert_array_equal(w, ww, err_msg=tag)
            np.testing.assert_array_equal(out, want, err_msg=tag)
        elif kind in ("identical", "underflow"):
            assert (w == w[0]).all(), f"{tag}: {w}"
            if kind == "identical":
                np.testing.assert_array_equal(out, c.X[0], err_msg=tag)
        else:
            want, ww = VO.aggregate(c.X.astype(f64), c.H, "gmed")
            close(out, want, rtol=0, atol=2e-5 * np.abs(c.X).max(), err_msg=tag)
            x0, v = c.X[0].astype(f64), (c.X[1].astype(f64) - c.X[0]) / 3
            s = float((out - x0) @ v / (v @ v))
            close(out, x0 + s * v, rtol=0, atol=2e-5 * np.abs(c.X).max(), err_msg=f"{tag}: off the line")


def test_nnm_exact_answers(K):
    """Every edge case: N_k by (D_kl, own row first, lower index) -- identical and underflowing rows: k, then the lowest
    indices; +inf distances: {k} alone; the mixed rows bitwise."""
    cases = EDGE + [E.identical(P, H=H) for P in (1, 1421) for H in (0, 5, 6)]
    cases = cases[:32]
    st = Stack(K, [c.X for c in cases])
    dst, wout = outputs(K, len(cases), 7), torch.full((len(cases), 60), NAN, device=K.dev)
    K.ops.nnm_mix([K.ops.vector_job(dst[j, OUT_OFF:], st.msgs, S, c.P, st.rows[j], c.H, K.L.MIX_NNM,
                                    weights_out=wout[j, W_OFF:]) for j, c in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, c in enumerate(cases):
        tag = f"nnm {c}"
        mixed, M = written(got[j], c.n, c.P, tag), wslice(gw[j], c.n * c.n, tag).reshape(c.n, c.n)
        sel, want = E.nnm(c)
        assert [list(np.flatnonzero(r > 0)) for r in M] == sel, tag
        for k in range(c.n):
            assert (M[k, sel[k]] == np.float32(1) / np.float32(len(sel[k]))).all(), tag
        np.testing.assert_array_equal(mixed, want, err_msg=tag)


def test_bucket_identical_rows(K):
    cases = [E.identical(P) for P in E.EDGE_P]
    st = Stack(K, [c.X for c in cases])
    jobs, spec = [], []
    dst = outputs(K, 12, 7)
    for j, (c, s) in enumerate((c, s) for c in cases for s in (1, 2, 3, 6)):
        jobs.append(K.ops.bucket_job(dst[j, OUT_OFF:], st.msgs, S, c.P, st.rows[cases.index(c)], s, seed=5, receiver=j))
        spec.append((c, s))
    K.ops.bucket_mix(jobs)
    got = dst.cpu().numpy()
    for j, (c, s) in enumerate(spec):
        rows = written(got[j], BO.n_out(c.n, s), c.P, f"bucket {c} s={s}")
        np.testing.assert_array_equal(rows, np.tile(c.X[0], (rows.shape[0], 1)))


MU_CASES = [c for c in EDGE if c.name.split("_")[0] in ("identical", "overflow", "underflow")]


def test_adaptive_attack_exact_answers(K):
    """P = 1, d = -sign(mu): min-max sends the honest extreme away from mu's sign, min-sum the header's
    sqrtf(n (c - sum e)) / n; identical rows and +inf / 0 distances: gamma = 0 and dst = mu, for every attack."""
    p1 = [[3, -1, 7, 5, 1], [-6, 2, -4, 0, -2, -8, 4]]
    blocks = [np.array(v, np.float32)[:, None] for v in p1] + [c.X for c in MU_CASES]
    st = Stack(K, blocks)
    jobs = [(0, "minmax_sgn"), (0, "minsum_sgn"), (1, "minmax_sgn"), (1, "minsum_sgn")]
    jobs += [(2 + i, AA.ATTACKS[(3 * i + q) % 6]) for i in range(len(MU_CASES)) for q in (0, 1)]
    dst, gam = outputs(K, len(jobs)), torch.full((len(jobs), 3), NAN, device=K.dev)
    K.ops.adaptive_attack([K.ops.adaptive_attack_job(dst[j, OUT_OFF:], st.msgs, S, blocks[b].shape[1], st.rows[b][:5],
                                                     a, 1.0, gamma_out=gam[j, 1:2]) for j, (b, a) in enumerate(jobs)])
    got, gg = dst.cpu().numpy(), gam.cpu().numpy()
    for j, (b, attack) in enumerate(jobs):
        P = blocks[b].shape[1]
        tag = f"{attack} block {b}"
        msg = written(got[j], 1, P, tag)[0]
        g = gg[j, 1]
        if b < 2:
            vals = p1[b][:5]
            if attack == "minmax_sgn":
                assert (g, msg[0]) == E.minmax_sgn_p1(vals), (tag, g, msg)
            else:
                g32, _, m32 = E.minsum_sgn_p1(vals)
                assert g == g32 and msg[0] == m32, (tag, g, msg, g32, m32)
        else:
            assert g == 0, tag
            np.testing.assert_array_equal(msg, E.f32_mean(blocks[b][:5]), err_msg=tag)


def test_tailored_and_pipeline_exact_answers(K):
    """Identical rows and +inf / 0 distances: gamma_mm = 0, so i* = 0, gamma_out = 0 and dst = mu; on identical rows
    the modelled aggregate is x itself, through every mixing and rule."""
    st = Stack(K, [c.X for c in MU_CASES])
    slots, honest = [0, 1, -1, 2, 3, -1, 4], [0, 1, 3, 4, 6]
    tjobs, pjobs = [], []
    for i, c in enumerate(MU_CASES):
        sl = [st.rows[i][s] if s >= 0 else -1 for s in slots]
        tjobs.append((c, sl, ("krum", "clip", "gmed", "mkrum")[i % 4], ("tailored_uv", "tailored_sgn")[i % 2]))
        for q, (rule, mixing) in enumerate((("dnc", None), ("mkrum", "nnm"), ("trim", ("bucket", 2)))):
            pjobs.append((c, sl, rule, mixing, ("pipeline_std", "pipeline_uv", "pipeline_sgn")[(i + q) % 3]))
    dst, gam = outputs(K, len(tjobs)), torch.full((len(tjobs), 2), NAN, device=K.dev)
    K.ops.tailored_attack([K.ops.tailored_attack_job(dst[j, OUT_OFF:], st.msgs, S, c.P, sl, honest, r, 1, a, 2.0,
                                                     gamma_out=gam[j, :1]) for j, (c, sl, r, a) in enumerate(tjobs)])
    got, gg = dst.cpu().numpy(), gam.cpu().numpy()
    for j, (c, sl, r, a) in enumerate(tjobs):
        tag = f"{a} {r} {c}"
        assert gg[j, 0] == 0 and np.isnan(gg[j, 1]), tag
        np.testing.assert_array_equal(written(got[j], 1, c.P, tag)[0], E.f32_mean(c.X[:5]), err_msg=tag)
    for g0 in range(0, len(pjobs), 16):
        part = pjobs[g0:g0 + 16]
        dst, gam, mod = outputs(K, len(part)), torch.full((len(part), 2), NAN, device=K.dev), outputs(K, len(part))
        K.ops.pipeline_attack([K.ops.pipeline_attack_job(dst[j, OUT_OFF:], st.msgs, S, c.P, sl, honest, r, 1, a, 2.0,
                                                         mixing=m, n_perms=3, seed=11, attacker=1, receiver=2,
                                                         gamma_out=gam[j, :1], model_out=mod[j, OUT_OFF:])
                               for j, (c, sl, r, m, a) in enumerate(part)])
        got, gg, mo = dst.cpu().numpy(), gam.cpu().numpy(), mod.cpu().numpy()
        for j, (c, sl, r, m, a) in enumerate(part):
            tag = f"{a} {r} {m} {c}"
            assert gg[j, 0] == 0 and np.isnan(gg[j, 1]), tag
            np.testing.assert_array_equal(written(got[j], 1, c.P, tag)[0], E.f32_mean(c.X[:5]), err_msg=tag)
            model = written(mo[j], 1, c.P, tag)[0]
            if c.name.startswith("identical"):
                np.testing.assert_array_equal(model, c.X[0], err_msg=tag)


def test_dissensus_exact_answers(K):
    cases = [E.line()] + [E.identical(P) for P in E.EDGE_P] + [E.scaled(P, E.OVER, "overflow") for P in E.EDGE_P]
    spec = [(c, n_byz, eps) for c in cases for n_byz, eps in ((1, 1.0), (2, 1.0), (4, 3.0), (2, 0.0))][:32]
    st = Stack(K, [c.X for c in cases])
    dst = outputs(K, len(spec))
    K.ops.dissensus_attack([K.ops.dissensus_attack_job(dst[j, OUT_OFF:], st.msgs, S, c.P, st.rows[cases.index(c)][0],
                                                       st.rows[cases.index(c)], n_byz, eps)
                            for j, (c, n_byz, eps) in enumerate(spec)])
    got = dst.cpu().numpy()
    for j, (c, n_byz, eps) in enumerate(spec):
        tag = f"dissensus {c} n_byz={n_byz} eps={eps}"
        out = written(got[j], 1, c.P, tag)[0]
        np.testing.assert_array_equal(out, E.dissensus(c, n_byz, eps), err_msg=tag)
        if eps == 0 or c.name.startswith("identical"):
            np.testing.assert_array_equal(out, c.X[0], err_msg=tag)


def test_mimic_exact_answers(K):
    """update 0 from z = 0: on a line the candidate furthest along sign(c_k0); identical rows and +inf / 0 norms: z
    stays 0, the lowest candidate is copied and reported."""
    cases = [c for c in EDGE if c.t is not None]
    spec = [(c, cand) for c in cases for cand in (list(range(7)), [1, 3, 5], [0, 1, 2, 3, 4, 5])][:32]
    st = Stack(K, [c.X for c in cases])
    dst = outputs(K, len(spec))
    zb = torch.full((len(spec), OUT_OFF + S), NAN, device=K.dev)
    for j, (c, _) in enumerate(spec):
        zb[j, OUT_OFF:OUT_OFF + c.P] = 0
    tgt = torch.full((len(spec), 3), -7, dtype=torch.int32, device=K.dev)
    K.ops.mimic_attack([K.ops.mimic_attack_job(dst[j, OUT_OFF:], st.msgs, S, c.P, st.rows[cases.index(c)], cand,
                                               zb[j, OUT_OFF:], 0, target_out=tgt[j, 1:2])
                        for j, (c, cand) in enumerate(spec)])
    got, zg, tg = dst.cpu().numpy(), zb.cpu().numpy(), tgt.cpu().numpy()
    for j, (c, cand) in enumerate(spec):
        tag = f"mimic {c} candidates={cand}"
        k, live = E.mimic(c, cand)
        assert tg[j, 1] == k and tg[j, 0] == -7 and tg[j, 2] == -7, (tag, tg[j])
        np.testing.assert_array_equal(written(got[j], 1, c.P, tag)[0], c.X[k], err_msg=tag)
        z = written(zg[j], 1, c.P, tag)[0]
        assert bool(z.any()) == live, tag


# ---------------------------------------------------------------------------------------------------------- d) API
@pytest.mark.parametrize("rule", ["krum", "mkrum", "scclip", "gmed", "dnc"])
@pytest.mark.parametrize("mixing", [None, "nnm", "bucket"])
def test_agent_api_on_one_and_six_parameters(K, rule, mixing):
    """RPBCAC_agent._resilient_aggregation on (n, 1) and (n, 2, 3) tensors: identical rows give x bitwise under every
    rule and mixing; the P = 1 line (no mixing) gives the closed form of the rule."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from golden_util import pretrained
    from test_aggregation_rules_gpu import build_models
    w, _, _ = pretrained()
    H = 1 if mixing == "bucket" and rule in ("krum", "mkrum") else 2        # 4 bucketed rows: krum needs H <= 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule,
                      mixing=mixing)
    for c in (E.identical(1), E.identical(6)):
        v = c.X.reshape((7, 1) if c.P == 1 else (7, 2, 3))
        got = np.asarray(ag._resilient_aggregation(v).numpy())
        assert got.shape == v.shape[1:]
        np.testing.assert_array_equal(got.reshape(-1), c.X[0], err_msg=f"{rule} {mixing} {c}")
    if mixing is None:
        c = E.line()
        want = {"krum": lambda: E.krum(c, "krum"), "mkrum": lambda: E.krum(c, "mkrum"), "scclip": lambda: E.scclip(c),
                "dnc": lambda: E.dnc(c), "gmed": lambda: VO.aggregate(c.X.astype(f64), 2, "gmed")[::-1]}[rule]()[1]
        got = np.asarray(ag._resilient_aggregation(c.X.reshape(7, 1)).numpy()).reshape(-1)
        if rule == "gmed":
            close(got, want, rtol=0, atol=2e-5 * 16)
        else:
            np.testing.assert_array_equal(got, want, err_msg=rule)
