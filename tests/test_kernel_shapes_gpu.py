"""GPU parity at the launch shapes the trainer uses: every kernel against the float64 oracle (oracle/rpbcac_oracle.py)
where the small shapes of test_kernels_gpu.py never go -- several 64-row chunks per grad warp, row windows and strided
targets, gathered rows, the job-count limits, several row-loop iterations per thread, the team kernel's neighbour-count
bounds, mixed consensus jobs, padded teams, non-square grids, unscaled states, split rollouts and episode means.

Row counts that must reach a code path are derived from the device's SM count.  Tolerances (SURVEY 8d): gradient sums
rtol 1e-4 with an atol floor growing with sqrt(B); forward values rtol 1e-5 / atol 3e-6 (5e-6 for sums of several
terms and for the clipped mean of neighbour estimates, as in test_kernels_gpu.py); weights after a projection or
consensus step rtol 1e-4 / atol 1e-6; discrete outputs exact.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from golden_util import pretrained                     # noqa: E402
from kernel_util import close, load_kernels, rand_net, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_S, IN_SA, IN_NS = 0, 1, 2          # rcmarl_input_kind (include/rcmarl.h)
MSE, CE = 0, 1                        # rcmarl_loss
CHUNK = 64                            # rows per grad warp chunk (TileLayout::ROWS, grad_kernel.cuh:43)
MAX_GRAD_WARPS = 8                    # upper bound of grad_warps (grad_kernel.cuh:86-98)
TAIL = 37                             # ragged last chunk
NROW = {5: 5, 16: 10}
ORACLE_CHUNK = 1 << 16


@pytest.fixture(scope="module")
def K():
    return load_kernels()


@pytest.fixture(scope="module")
def SMS(K):
    return torch.cuda.get_device_properties(0).multi_processor_count


class Buf:
    """Seeded buffer rows (time-major, row = t * n_envs + e) on the host (flattened per input kind) and the device."""

    def __init__(self, K, rs, NA, n):
        s, ns, a, r = synth(rs, n, NA, NROW[NA])
        self.NA, self.n = NA, n
        self.x = {IN_S: s.reshape(n, -1), IN_SA: np.concatenate([s, a], -1).reshape(n, -1), IN_NS: ns.reshape(n, -1)}
        self.a, self.r = a[:, :, 0], r[:, :, 0]
        self.dsa, self.dns, self.dr = to_dev(K, self.x[IN_SA], self.x[IN_NS], self.r)

    def rows(self, K, **kw):
        return K.ops.make_rows(self.dsa, self.dns, self.dr, self.NA, **kw)


def d_in(NA, kind):
    return 3 * NA if kind == IN_SA else 2 * NA


def fwd(w, X):
    """fp64 network output over the rows of X (float32, any length), ORACLE_CHUNK rows at a time."""
    w64 = O.cast_weights(w, f64)
    return np.concatenate([O.mlp_forward(w64, X[lo:lo + ORACLE_CHUNK].astype(f64))
                           for lo in range(0, len(X), ORACLE_CHUNK)])


def oracle_mse_sums(w, X, idx, y):
    """[sum_rows e * dout/dtheta | sum_rows e^2] over the rows idx of X, e = net(x) - y (what rcmarl_grad returns)."""
    w64 = O.cast_weights(w, f64)
    g_tot, l_tot = 0.0, 0.0
    for lo in range(0, len(idx), ORACLE_CHUNK):
        out, cch = O.mlp_forward(w64, X[idx[lo:lo + ORACLE_CHUNK]].astype(f64), cache=True)
        e = out - y[lo:lo + ORACLE_CHUNK].astype(f64).reshape(-1, 1)
        g_tot = g_tot + np.concatenate([t.reshape(-1) for t in O.mlp_backward(w64, cch, e)])
        l_tot += float((e * e).sum())
    return g_tot, l_tot


def oracle_ce_sums(w, X, idx, act, d):
    """[sum_rows d * dCE/dtheta | sum_rows d * CE] with CE = -log softmax(net(x))[act] (actor_ce_step without the 1/B)."""
    w64 = O.cast_weights(w, f64)
    g_tot, l_tot = 0.0, 0.0
    for lo in range(0, len(idx), ORACLE_CHUNK):
        logits, cch = O.mlp_forward(w64, X[idx[lo:lo + ORACLE_CHUNK]].astype(f64), cache=True)
        lsm = O.log_softmax(logits)
        ai = act[lo:lo + ORACLE_CHUNK].astype(np.int64)
        dd = d[lo:lo + ORACLE_CHUNK].astype(f64)
        ar = np.arange(len(ai))
        l_tot += float((dd * -lsm[ar, ai]).sum())
        p = np.exp(lsm)
        p[ar, ai] -= 1.0
        g_tot = g_tot + np.concatenate([t.reshape(-1) for t in O.mlp_backward(w64, cch, p * dd[:, None])])
    return g_tot, l_tot


# ---------------------------------------------------------------------------------------------------------- grad helpers
def grad_ctas(K, NA, kinds, loss, n_rows, sms):
    """CTAs per job of rcmarl_grad's one-wave grid (equal shares), from the library's own plan."""
    n = len(kinds)
    out = (C.c_int32 * n)()
    K.L.check(K.L.lib().rcmarl_grad_grid_plan(NA, (C.c_int32 * n)(*kinds), n, loss, n_rows, 0, sms, out),
              "rcmarl_grad_grid_plan")
    return list(out)


def steady_rows(K, NA, kinds, loss, sms):
    """Rows for which every warp of every job sweeps at least 3 full 64-row chunks, plus a ragged tail of TAIL rows."""
    full = 3 * max(1, sms // len(kinds)) * MAX_GRAD_WARPS
    B = full * CHUNK + TAIL
    ctas = grad_ctas(K, NA, kinds, loss, B, sms)
    assert all(B // CHUNK >= 3 * c * MAX_GRAD_WARPS for c in ctas), (B, ctas)
    assert B % CHUNK != 0
    return B


def grad_spec(K, rs, buf, loss, kind, j, idx, strided=False, time_idx=None):
    """One grad job over the absolute rows idx.  strided: the target is the column view r[:, i] (target_stride = NA)."""
    NA = buf.NA
    net = rand_net(rs, 2 * NA, 5) if loss == CE else rand_net(rs, d_in(NA, kind), 1)
    if strided:
        col = (j + 1) % NA
        tgt, tgt_dev, stride = buf.r[:, col], buf.dr[:, col], NA
    else:
        tgt = ((1.0 + 0.5 * j) * rs.randn(buf.n)).astype(np.float32)     # distinct target / TD-error weights per job
        tgt_dev, stride = to_dev(K, tgt)[0], 1
    return dict(kind=kind, net=net, w=to_dev(K, K.nets.pack(net))[0], tgt=tgt, tgt_dev=tgt_dev, stride=stride,
                agent=j % NA if loss == CE else 0, time_idx=time_idx, idx=idx)


def grad_jobs(K, specs):
    """Job structs and NaN-filled [grad | loss] sums (the reduction must write every entry)."""
    jobs, sums = [], []
    for sp in specs:
        s = torch.full((sp["w"].numel() + 1,), NAN, device=K.dev)
        jobs.append(K.ops.grad_job(sp["w"], sp["tgt_dev"], s, sp["kind"], action_agent=sp["agent"],
                                   target_stride=sp["stride"], time_idx=sp["time_idx"]))
        sums.append(s)
    return jobs, sums


def check_grad(buf, loss, specs, sums):
    for j, (sp, got) in enumerate(zip(specs, sums)):
        idx = sp["idx"]
        y = sp["tgt"][idx]
        if loss == MSE:
            g, l = oracle_mse_sums(sp["net"], buf.x[sp["kind"]], idx, y)
        else:
            g, l = oracle_ce_sums(sp["net"], buf.x[IN_S], idx, buf.a[idx, sp["agent"]], y)
        got = got.cpu().numpy()
        atol = 2e-6 * max(1.0, np.abs(g).max()) * max(1, len(idx)) ** 0.5
        close(got[:-1], g, rtol=1e-4, atol=atol, err_msg=f"gradient of job {j} (kind {sp['kind']})")
        if loss == MSE:                                   # sum of squares: no cancellation
            close(got[-1], l, rtol=1e-5, atol=1e-6, err_msg=f"loss of job {j}")
        else:                                             # signed TD-error weights: a cancelling sum like the gradient
            close(got[-1], l, rtol=1e-4, atol=atol, err_msg=f"loss of job {j}")


def run_and_check_grad(K, buf, rows, loss, specs):
    jobs, sums = grad_jobs(K, specs)
    K.ops.grad(rows, jobs, loss)
    check_grad(buf, loss, specs, sums)


# ---------------------------------------------------------------------------------------------------------- 1. grad steady state
STEADY = {
    "mse5_one_job": (5, MSE, [IN_S]),
    "mse5_fit_first_8_jobs": (5, MSE, [IN_SA, IN_S] * 4),       # the trainer's fit_first: TR (sa) + critic (s) per agent
    "mse16_three_kinds": (16, MSE, [IN_S, IN_SA, IN_NS]),
    "ce5_four_agents": (5, CE, [IN_S] * 4),
    "ce16_four_agents": (16, CE, [IN_S] * 4),
}


@pytest.mark.parametrize("case", list(STEADY))
def test_grad_steady_state_sweep_matches_oracle(K, SMS, case):
    """GradCore::sweep steady state (grad_kernel.cuh:244-401): every warp sweeps >= 3 chunks (c += cstep), accumulating
    in registers across chunks; at NA = 5 every full chunk is bulk-copied (the mbarrier phase flips, :259-260, and the
    prefetch of the next chunk, :273-281) and the ragged last chunk falls back to per-lane loads (stage_src, :222-226);
    at NA = 16 all chunks use per-lane loads.  CE: the action read from sa (:321) per job's action_agent."""
    NA, loss, kinds = STEADY[case]
    B = steady_rows(K, NA, kinds, loss, SMS)
    rs = np.random.RandomState(100 + len(kinds) + NA + 7 * loss)
    buf = Buf(K, rs, NA, B)
    idx = np.arange(B)
    specs = [grad_spec(K, rs, buf, loss, kind, j, idx) for j, kind in enumerate(kinds)]
    run_and_check_grad(K, buf, buf.rows(K), loss, specs)


# ---------------------------------------------------------------------------------------------------------- 2. row windows
@pytest.mark.parametrize("NA,row_begin", [(5, 64 * 7), (5, 64 * 7 + 1), (16, 64 * 7 + 1)])
@pytest.mark.parametrize("loss", [MSE, CE])
def test_grad_row_window_and_strided_target(K, SMS, NA, row_begin, loss):
    """Contiguous rows [row_begin, row_begin + n) with column-view targets r[:, i], target_stride = NA
    (grad_kernel.cuh:306, trainer.py:297) and, for CE, the actor window (trainer.py:361-383) reading the action from sa
    (:321).  At NA = 5 the alignment test in stage_src (grad_kernel.cuh:222-226) picks bulk-copy staging when
    row_begin is a multiple of 64 (16-byte aligned sa / ns spans) and per-lane loads when it is odd."""
    kinds = [IN_S, IN_SA, IN_NS] if loss == MSE else [IN_S] * 3
    n = steady_rows(K, NA, kinds, loss, SMS)
    aligned = all((row_begin * f * 4) % 16 == 0 for f in (3 * NA, 2 * NA))
    assert aligned == (row_begin % 2 == 0 or NA == 16)
    rs = np.random.RandomState(200 + row_begin + NA + loss)
    buf = Buf(K, rs, NA, row_begin + n + 101)            # rows after the window must not be read either
    idx = np.arange(row_begin, row_begin + n)
    specs = [grad_spec(K, rs, buf, loss, kind, j, idx, strided=True) for j, kind in enumerate(kinds)]
    run_and_check_grad(K, buf, buf.rows(K, row_begin=row_begin, n_rows=n), loss, specs)


# ---------------------------------------------------------------------------------------------------------- 3. gathered rows
@pytest.mark.parametrize("N", [24, 64, 96, 128])
@pytest.mark.parametrize("loss", [MSE, CE])
def test_grad_gathered_rows_per_job_time_idx(K, N, loss):
    """Gathered mode, row(m) = row_begin + time_idx[m / N] * N + m % N (common.cuh:47-51), with a different per-job
    time_idx override for each of 4 jobs (grad_kernel.cuh:464) and row_begin = k * N, as the adversaries' actor
    mini-batches run (trainer.py:431-447).  N % 64 == 0 takes the bulk-copy gather (gather_ok, grad_kernel.cuh:221),
    N = 24 / 96 per-lane loads."""
    NA, T_buf, k, Tm = 5, 240, 17, 201
    rs = np.random.RandomState(300 + N + loss)
    buf = Buf(K, rs, NA, T_buf * N)
    row_begin = k * N
    tables = np.stack([rs.permutation(T_buf - k)[:Tm] for _ in range(5)]).astype(np.int32)
    dtab = to_dev(K, tables)[0]
    kinds = [IN_S, IN_SA, IN_NS, IN_SA] if loss == MSE else [IN_S] * 4
    specs = [grad_spec(K, rs, buf, loss, kind, j, row_begin + O.expand_time_perm(tables[j], N), strided=(j % 2 == 0),
                       time_idx=dtab[j]) for j, kind in enumerate(kinds)]
    rows = buf.rows(K, row_begin=row_begin, time_idx=dtab[4], n_envs=N)     # the row set's own table: overridden by every job
    assert rows.n_rows == Tm * N
    run_and_check_grad(K, buf, rows, loss, specs)


# ---------------------------------------------------------------------------------------------------------- 4. job-count edges
def test_grad_32_jobs_and_33_rejected(K, SMS):
    """RCMARL_MAX_JOBS grad jobs in one launch: a 16-agent all-cooperative team's fit (16 x {IN_S, IN_SA}), CTA ranges
    through the int16 cta_first (grad_kernel.cuh:134, :484-486; plan_grid, train_kernels.cu); 33 jobs are
    refused (rcmarl_grad, train_kernels.cu)."""
    NA = 16
    kinds = [IN_S, IN_SA] * 16
    B = steady_rows(K, NA, kinds, MSE, SMS)
    rs = np.random.RandomState(400)
    buf = Buf(K, rs, NA, B)
    idx = np.arange(B)
    specs = [grad_spec(K, rs, buf, MSE, kind, j, idx, strided=(j % 3 == 0)) for j, kind in enumerate(kinds)]
    rows = buf.rows(K)
    run_and_check_grad(K, buf, rows, MSE, specs)
    jobs, _ = grad_jobs(K, specs + specs[:1])
    with pytest.raises(K.L.RcmarlError):
        K.ops.grad(rows, jobs, MSE)


def test_values_32_jobs(K):
    """RCMARL_MAX_JOBS value jobs in one launch (blockIdx.y = job, train_kernels.cu:62): 1-3 terms of every kind with
    distinct scales, optional strided additive column, and an actor softmax job."""
    NA, B, gamma = 16, 3001, 0.9
    rs = np.random.RandomState(401)
    buf = Buf(K, rs, NA, B)
    nets = {kind: [rand_net(rs, d_in(NA, kind), 1) for _ in range(3)] for kind in (IN_S, IN_SA, IN_NS)}
    dnets = {kind: [to_dev(K, K.nets.pack(w))[0] for w in ws] for kind, ws in nets.items()}
    wa = rand_net(rs, 2 * NA, 5)
    jobs, outs, wants = [], [], []
    for j in range(31):
        terms, want = [], np.zeros(B)
        for t in range(1 + j % 3):
            kind, m, scale = (j + t) % 3, (j + 2 * t) % 3, [1.0, gamma, -1.0][t] * (1 + 0.1 * j)
            terms.append((dnets[kind][m], kind, scale))
            want += np.float32(scale) * fwd(nets[kind][m], buf.x[kind])[:, 0]
        add = dict(add=buf.dr, add_stride=NA, add_off=j % NA, add_scale=0.5 + 0.05 * j) if j % 2 == 0 else {}
        if add:
            want += np.float32(add["add_scale"]) * buf.r[:, j % NA].astype(f64)
        out = torch.full((B,), NAN, device=K.dev)
        jobs.append(K.ops.value_job(out, terms, **add))
        outs.append(out)
        wants.append(want)
    probs = torch.full((B, 5), NAN, device=K.dev)
    jobs.append(K.ops.value_job(probs, [(to_dev(K, K.nets.pack(wa))[0], IN_NS, 1.0)], n_out=5, softmax=1))
    K.ops.values(buf.rows(K), jobs)
    for j, (out, want) in enumerate(zip(outs, wants)):
        close(out, want, rtol=1e-5, atol=5e-6, err_msg=f"value job {j}")
    close(probs, O.softmax(fwd(wa, buf.x[IN_NS])), rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------- team helpers
def oracle_team(own, heads, X, H):
    """fp64 clipped mean of the neighbour-head estimates and the projection sums
    [sum c * phi (20) | sum c | sum (agg - pred) * c], c = (agg - pred) / (||phi||^2 + 1)."""
    w64 = O.cast_weights(own, f64)
    phi = O.mlp_features(w64, X.astype(f64))
    est = np.stack([(phi @ m[4].astype(f64) + m[5].astype(f64))[:, 0] for m in heads])
    agg = O.resilient_aggregation(est, H)
    err = agg - (phi @ w64[4] + w64[5])[:, 0]
    c = err / ((phi * phi).sum(1) + 1.0)
    return agg, np.concatenate([phi.T @ c, [c.sum(), (err * c).sum()]])


def run_team(K, rs, buf, cfg, B):
    """cfg: list of (kind, n_in, H).  Every job has its own network and neighbours drawn from a 16-message stack of its
    kind.  Returns the per-job data, NaN-prefilled sums and agg_out after one rcmarl_team call."""
    NA = buf.NA
    msgs = {kind: [rand_net(rs, d_in(NA, kind), 1) for _ in range(16)] for kind in (IN_S, IN_SA)}
    dmsgs = {kind: to_dev(K, np.stack([K.nets.pack(w) for w in ws]))[0] for kind, ws in msgs.items()}
    jobs, data = [], []
    for kind, n_in, H in cfg:
        own = rand_net(rs, d_in(NA, kind), 1)
        nodes = [int(v) for v in rs.permutation(16)[:n_in]]
        dw = to_dev(K, K.nets.pack(own))[0]
        sums = torch.full((22,), NAN, device=K.dev)
        agg = torch.full((buf.n,), NAN, device=K.dev)
        P = K.L.param_count(d_in(NA, kind), 1)
        jobs.append(K.ops.team_job(dw, kind, dmsgs[kind], P, nodes, H, sums=sums, agg_out=agg))
        data.append(dict(kind=kind, H=H, own=own, dw=dw, P=P, heads=[msgs[kind][i] for i in nodes], sums=sums, agg=agg))
    K.ops.team(buf.rows(K, n_rows=B), jobs)
    return data


def check_team(buf, data, B):
    for j, d in enumerate(data):
        agg, sums = oracle_team(d["own"], d["heads"], buf.x[d["kind"]][:B], d["H"])
        close(d["agg"][:B], agg, rtol=1e-5, atol=5e-6, err_msg=f"agg_out of team job {j}")
        assert torch.isnan(d["agg"][B:]).all()
        scale = max(1.0, np.abs(sums[:21]).max())
        close(d["sums"], sums, rtol=1e-4, atol=2e-6 * scale * B ** 0.5, err_msg=f"sums of team job {j}")
        d["want_agg"] = agg


@pytest.mark.parametrize("NA,n_agents", [(5, 4), (16, 16)])
def test_team_many_jobs(K, NA, n_agents):
    """rcmarl_team with 8 jobs (4 agents x {critic, TR}) and with 32 jobs at NA = 16: one launch per input kind through
    job_list (train_kernels.cu:770-794), partials written [y][job] interleaved (:309) and reduced with step n_jobs (:797)."""
    rs = np.random.RandomState(410 + NA)
    B = 4001
    buf = Buf(K, rs, NA, B + 50)
    cfg = []
    for _ in range(n_agents):
        n_in = int(rs.randint(1, 17))
        H = int(rs.randint(0, min(7, n_in - 1) + 1))
        cfg += [(IN_S, n_in, H), (IN_SA, n_in, H)]
    check_team(buf, run_team(K, rs, buf, cfg, B), B)


# ---------------------------------------------------------------------------------------------------------- 5. values loop
@pytest.mark.parametrize("NA", [5, 16])
def test_values_several_iterations_per_thread(K, SMS, NA):
    """values_kernel's two-rows-per-iteration loop (train_kernels.cu:90-114) over an odd number (>= 3) of grid passes,
    so that the second row of the last pair is dead, and the single-row actor softmax loop (:66-83); rows in a window
    [row_begin, row_begin + B): nothing outside it is written."""
    pass_rows = 2 * SMS * 256                         # one pass of the one-wave grid (launch_values, :407-410)
    B = 2 * pass_rows + pass_rows // 2 + 37
    stride = min(-(-B // 256), 2 * SMS) * 256
    n_iter = -(-B // stride)
    assert n_iter >= 3 and n_iter % 2 == 1, n_iter
    rs = np.random.RandomState(500 + NA)
    row_begin, gamma = 1001, 0.9
    buf = Buf(K, rs, NA, row_begin + B + 300)
    wc, wt, wa = rand_net(rs, 2 * NA, 1), rand_net(rs, 3 * NA, 1), rand_net(rs, 2 * NA, 5)
    dwc, dwt, dwa = to_dev(K, K.nets.pack(wc), K.nets.pack(wt), K.nets.pack(wa))
    td_err = torch.full((buf.n,), NAN, device=K.dev)
    td_tgt = torch.full((buf.n,), NAN, device=K.dev)
    probs = torch.full((buf.n, 5), NAN, device=K.dev)
    K.ops.values(buf.rows(K, row_begin=row_begin, n_rows=B), [
        K.ops.value_job(td_err, [(dwt, IN_SA, 1.0), (dwc, IN_NS, gamma), (dwc, IN_S, -1.0)]),
        K.ops.value_job(td_tgt, [(dwc, IN_NS, gamma)], add=buf.dr, add_stride=NA, add_off=2),
        K.ops.value_job(probs, [(dwa, IN_S, 1.0)], n_out=5, softmax=1)])
    w = slice(row_begin, row_begin + B)
    V, nV = fwd(wc, buf.x[IN_S][w])[:, 0], fwd(wc, buf.x[IN_NS][w])[:, 0]
    TR = fwd(wt, buf.x[IN_SA][w])[:, 0]
    close(td_err[w], TR + np.float32(gamma) * nV - V, rtol=1e-5, atol=5e-6)
    close(td_tgt[w], buf.r[w, 2].astype(f64) + np.float32(gamma) * nV, rtol=1e-5, atol=3e-6)
    close(probs[w], O.softmax(fwd(wa, buf.x[IN_S][w])), rtol=1e-5, atol=1e-6)
    for t in (td_err, td_tgt, probs):
        assert torch.isnan(t[:row_begin]).all() and torch.isnan(t[row_begin + B:]).all()


# ---------------------------------------------------------------------------------------------------------- 6. team loop, MAXN
@pytest.mark.parametrize("NA", [5, 16])
def test_team_several_iterations_and_neighbour_bounds(K, SMS, NA):
    """team_body's two-rows-per-iteration loop (train_kernels.cu:239-295) over an odd number (>= 3) of passes for both
    input kinds, with n_in on both sides of the MAXN switch points (4 | 5 and 8 | 9, :318-324) and H up to 7; the
    projected output layers after rcmarl_sgd_apply against critic_update_team / TR_update_team."""
    cfg_c = [(4, 3), (5, 2), (8, 7), (9, 4), (16, 7)]
    cfg_t = [(4, 1), (5, 4), (8, 3), (9, 7), (16, 5)]
    n_list = len(cfg_c)                                   # jobs per input kind = per launch
    cap = max(1, (SMS * 3) // n_list)                     # grid_y_for (train_kernels.cu:485-492), 3 CTAs per SM
    B = 2 * cap * 128 + cap * 64 + 37
    gy = min(-(-B // 256), cap)
    n_iter = -(-B // (gy * 128))
    assert n_iter >= 3 and n_iter % 2 == 1, n_iter
    rs = np.random.RandomState(600 + NA)
    buf = Buf(K, rs, NA, B)
    cfg = [(IN_S, n, H) for n, H in cfg_c] + [(IN_SA, n, H) for n, H in cfg_t]
    data = run_team(K, rs, buf, cfg, B)
    check_team(buf, data, B)
    new = [d["dw"].clone() for d in data]
    K.ops.sgd_apply([K.ops.sgd_job(nw, d["dw"], d["sums"], d["P"], -1.0 / B, first=d["P"] - 21) for nw, d in zip(new, data)])
    for j, (nw, d) in enumerate(zip(new, data)):
        dummy = rand_net(rs, 2 * NA, 5)
        if d["kind"] == IN_S:
            ag = O.RPBCACOracleAgent(dummy, d["own"], rand_net(rs, 3 * NA, 1), 0.002, 0.01, H=d["H"], dtype=f64)
            ag.critic_update_team(buf.x[IN_S], d["want_agg"])
            want = ag.critic
        else:
            ag = O.RPBCACOracleAgent(dummy, rand_net(rs, 2 * NA, 1), d["own"], 0.002, 0.01, H=d["H"], dtype=f64)
            ag.TR_update_team(buf.x[IN_SA], d["want_agg"])
            want = ag.TR
        close(nw, K.nets.pack(want), rtol=1e-4, atol=1e-6, err_msg=f"projected weights of team job {j}")


# ---------------------------------------------------------------------------------------------------------- 7. consensus
@pytest.mark.parametrize("NA", [5, 16])
def test_consensus_hidden_critic_and_tr_jobs(K, NA):
    """consensus_hidden_kernel (train_kernels.cu:331-340) as the trainer launches it (trainer.py:325-326): critic and
    TR jobs of different n_hidden in one call (job 0 a critic, the TR jobs set the grid), n_in 1..16 with repeated
    in_nodes, H up to 7, up to 32 jobs; the output layers stay bitwise untouched."""
    rs = np.random.RandomState(700 + NA)
    n_ag = NA
    dims = {IN_S: 2 * NA, IN_SA: 3 * NA}
    nets = {k: [rand_net(rs, dims[k], 1) for _ in range(n_ag)] for k in dims}
    msgs = {k: to_dev(K, np.stack([K.nets.pack(w) for w in nets[k]]))[0] for k in dims}
    own = {k: [rand_net(rs, dims[k], 1) for _ in range(n_ag)] for k in dims}
    dst = {k: to_dev(K, np.stack([K.nets.pack(w) for w in own[k]]))[0] for k in dims}
    before = {k: v.clone() for k, v in dst.items()}
    nh = {k: K.nets.n_hidden_params(dims[k]) for k in dims}
    assert nh[IN_S] < nh[IN_SA]
    jobs, cfg = [], []
    for i in range(n_ag):
        for k, n_in in ((IN_S, 1 + (7 * i) % 16), (IN_SA, 16 - (7 * i) % 16)):
            nodes = [i] + [int(v) for v in rs.randint(0, n_ag, size=n_in - 1)]      # own first, repeats allowed
            H = int(rs.randint(0, min(7, n_in - 1) + 1))
            jobs.append(K.ops.consensus_job(dst[k][i], msgs[k], msgs[k].shape[1], nh[k], nodes, H))
            cfg.append((k, i, nodes, H))
    assert len(jobs) == 2 * n_ag and cfg[0][0] == IN_S
    K.ops.consensus_hidden(jobs)
    for k, i, nodes, H in cfg:
        ag = O.RPBCACOracleAgent(rand_net(rs, 2 * NA, 5), own[IN_S][i], own[IN_SA][i], 0.002, 0.01, H=H, dtype=f64)
        if k == IN_S:
            ag.resilient_consensus_critic_hidden([nets[k][m] for m in nodes])
            want = ag.critic
        else:
            ag.resilient_consensus_TR_hidden([nets[k][m] for m in nodes])
            want = ag.TR
        close(dst[k][i], K.nets.pack(want), rtol=1e-4, atol=1e-6, err_msg=f"kind {k} agent {i} n_in {len(nodes)} H {H}")
        assert torch.equal(dst[k][i][nh[k]:], before[k][i][nh[k]:])


# ---------------------------------------------------------------------------------------------------------- 8. rollout
def rollout_parity(K, rs, NA, nact, nrow, ncol, scaling=True, N=32, n_ep=6, L_=20, gamma=0.9):
    """rcmarl_rollout with injected randomness against O.rollout_block on the unpadded nact-agent problem; slots of
    absent agents (nact .. NA-1) must be written as exact zeros.  Episodes where a uniform sits within fp32 noise of a
    CDF edge (a 'tie') are masked as in test_rollout_matches_oracle_with_injected_randomness."""
    actors = [rand_net(rs, 2 * nact, 5) for _ in range(nact)]
    critics = [rand_net(rs, 2 * nact, 1) for _ in range(nact)]
    desired = np.stack([rs.randint(0, nrow, nact), rs.randint(0, ncol, nact)], -1)
    init = np.stack([rs.randint(0, nrow, (n_ep, N, nact)), rs.randint(0, ncol, (n_ep, N, nact))], -1).astype(np.int32)
    init[0, 0] = desired                                  # start on the goal: reward-0 branch
    U = rs.rand(n_ep, L_, N, nact, 3).astype(np.float32)
    agents = [O.RPBCACOracleAgent(actors[i], critics[i], rand_net(rs, 3 * nact, 1), 0.002, 0.01, gamma, dtype=f64)
              for i in range(nact)]
    env = O.GridWorldOracle(nrow, ncol, nact, desired, n_envs=N, scaling=scaling)
    S, NS_, A, R, est, ret = O.rollout_block(env, agents, ['Cooperative'] * nact, n_episodes=n_ep, max_ep_len=L_,
                                             gamma=gamma, init_states=init, uniforms=U)
    pa = [K.nets.pack_padded(w, 2 * NA) for w in actors] + [K.nets.pack(rand_net(rs, 2 * NA, 5)) for _ in range(NA - nact)]
    pc = [K.nets.pack_padded(w, 2 * NA) for w in critics] + [K.nets.pack(rand_net(rs, 2 * NA, 1)) for _ in range(NA - nact)]
    des = np.zeros((NA, 2), np.int32)
    des[:nact] = desired
    T = n_ep * L_
    dsa, dns, dr = (torch.full((T * N, f * NA), NAN, device=K.dev) for f in (3, 2, 1))
    dest, dret = (torch.full((n_ep, N, NA), NAN, device=K.dev) for _ in range(2))
    aw, cw, ddes, dinit, dU = to_dev(K, np.stack(pa), np.stack(pc), des, init, U)
    K.ops.rollout(aw, cw, ddes, dsa, dns, dr, 0, dest, dret, n_envs=N, n_agents=NA, n_episodes=n_ep, max_ep_len=L_,
                  nrow=nrow, ncol=ncol, gamma=gamma, mu=0.1, uniforms=dU, init_state=dinit, scaling=scaling,
                  n_active=nact)
    got_sa = dsa.cpu().numpy().reshape(T * N, NA, 3)
    got_ns = dns.cpu().numpy().reshape(T * N, NA, 2)
    got_r, got_est, got_ret = dr.cpu().numpy(), dest.cpu().numpy(), dret.cpu().numpy()
    for x in (got_sa[:, nact:], got_ns[:, nact:], got_r[:, nact:], got_est[..., nact:], got_ret[..., nact:]):
        assert np.array_equal(x, np.zeros_like(x))        # absent agents: exact zeros (NaN-prefilled buffers)
    act_equal = got_sa[:, :nact, 2] == A[:, :, 0]
    assert act_equal.mean() > 0.999, act_equal.mean()
    ok_ep = np.ones((n_ep, N), bool)
    for row, _ag in np.argwhere(~act_equal):
        t, e = divmod(row, N)
        ok_ep[t // L_, e] = False
    assert ok_ep.mean() > 0.9
    mask = np.repeat(ok_ep, L_, axis=0).reshape(-1)
    assert np.array_equal(got_sa[mask][:, :nact, :2], S.astype(np.float32)[mask])
    assert np.array_equal(got_ns[mask][:, :nact], NS_.astype(np.float32)[mask])
    assert np.array_equal(got_r[mask][:, :nact], R.astype(np.float32)[mask][:, :, 0])
    close(got_est[..., :nact][ok_ep], est[ok_ep], rtol=1e-5, atol=3e-6)
    close(got_ret[..., :nact][ok_ep], ret[ok_ep], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("NA,nact,nrow", [(5, 3, 5), (16, 8, 10)])
def test_rollout_padded_team(K, NA, nact, nrow):
    """rollout_kernel with n_active < n_agents (rollout_consensus.cu:347-433): a team of n_active agents on the next
    kernel instantiation, weights padded with nets.pack_padded (main.py --n_agents other than 5 or 16)."""
    rollout_parity(K, np.random.RandomState(800 + nact), NA, nact, nrow, nrow)


@pytest.mark.parametrize("nrow,ncol", [(4, 6), (6, 4)])
def test_rollout_non_square_grid(K, nrow, ncol):
    """Non-square grids: resets draw y from [0, ncol) (rollout_consensus.cu:364-365), moves clip both coordinates with
    nrow - 1 (agent_step, :271-279, grid_world.py:55), and y is scaled with the y axis' own mean / std over
    max(nrow, ncol) table entries (ops.state_tables)."""
    rollout_parity(K, np.random.RandomState(810 + nrow), 5, 5, nrow, ncol)


def test_rollout_unscaled_states(K):
    """scaling=False (the reference Grid_World default): the network inputs and the sa / ns rows come from identity
    state tables (rollout_consensus.cu:371-372, :422-423; ops.state_tables)."""
    rollout_parity(K, np.random.RandomState(820), 5, 5, 5, 5, scaling=False)


def test_rollout_split_by_episode_offset_is_bitwise_equal(K):
    """Philox streams keyed by (seed, env, episode_offset + episode, step, agent) (rollout_consensus.cu:341-343, :362,
    :407) and rows placed by time_begin (:390): one call of 10 episodes equals two calls of 5, the second with
    episode_offset = 5 and time_begin = 5 * max_ep_len, bit for bit."""
    NA, N, n_ep, L_ = 5, 96, 10, 20
    w, desired, _ = pretrained()
    aw, cw = to_dev(K, np.stack([K.nets.pack(w[i][0]) for i in range(NA)]), np.stack([K.nets.pack(w[i][1]) for i in range(NA)]))
    ddes = to_dev(K, np.asarray(desired, np.int32))[0]
    T = n_ep * L_

    def buffers():
        return ([torch.full((T * N, f * NA), NAN, device=K.dev) for f in (3, 2, 1)],
                [torch.full((n_ep, N, NA), NAN, device=K.dev) for _ in range(2)])

    def run(bufs, logs, ep0, n):
        K.ops.rollout(aw, cw, ddes, *bufs, ep0 * L_, *logs, n_envs=N, n_agents=NA, n_episodes=n, max_ep_len=L_, nrow=5,
                      ncol=5, gamma=0.9, seed=0x5EED1234ABCD, episode_offset=ep0)
    one, one_log = buffers()
    run(one, one_log, 0, n_ep)
    two, two_log = buffers()
    h = n_ep // 2
    run(two, [x[:h] for x in two_log], 0, h)
    run(two, [x[h:] for x in two_log], h, n_ep - h)
    for a, b in zip(one + one_log, two + two_log):
        assert not torch.isnan(a).any()
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------- 9. episode means
@pytest.mark.parametrize("n_envs", [1, 255, 256, 257, 4096])
@pytest.mark.parametrize("NA", [5, 16])
def test_episode_means_match_fp64(K, n_envs, NA):
    """episode_mean_kernel (rollout_consensus.cu:438-452): per-thread serial sums over e = tid, tid + 256, ..., a fixed
    256-wide tree, one division.  Every input passes through at most ceil(n/256) - 1 + 8 additions, so the fp32 mean is
    within (ceil(n/256) + 8) * 2^-24 * max|x| of the exact one (first order) plus the rounding of the quotient."""
    rs = np.random.RandomState(900 + n_envs + NA)
    n_ep = 3
    x = (3.0 * rs.randn(n_ep, n_envs, NA) - 1.0).astype(np.float32)
    got = K.ops.episode_means(to_dev(K, x)[0])
    depth = -(-n_envs // 256) + 8
    close(got, x.astype(f64).mean(1), rtol=1e-6, atol=depth * 2.0 ** -24 * np.abs(x).max())
