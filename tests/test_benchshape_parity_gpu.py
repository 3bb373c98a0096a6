"""Oracle parity AT THE BENCHMARKED SHAPES (one GPU):
 (a) a Malicious + cooperative update round through rcmarl.trainer.Trainer with n_envs in {64, 128, 4096}: gathered row
     mode with n_envs % 64 == 0, i.e. the bulk-copy (TMA) staging branch of grad_kernel and the persistent mini-batch
     kernel (rcmarl_minibatch_fit) that the C2 benchmark spends half of its step in, at 4096 on the C2 grid (more than 32
     CTAs per chain); and the mixed team [Cooperative, Malicious, Greedy, Cooperative, Malicious] at n_envs = 1024, whose
     8 chains share one launch -- against the fp64 oracle;
 (b) rcmarl_grad over 4.1 M buffer rows (the C2 row count of one block) against NumPy fp64 sums (chunked);
 (c) rcmarl_clip_mean on the C5 tensor (64 x 1 048 576), H in {0, 1, 2, 4}, against oracle.resilient_aggregation;
 (d) the reference's own train_RPBCAC run with a Greedy and a Faulty agent and common_reward=True
     (tests/golden/ref_adversaries.npz, recorded by oracle/make_golden.py from the reference sources) through Trainer.
Tolerances as in the other GPU tests: gradient sums rtol 1e-4 (+ a sqrt(B) fp32 accumulation floor), weights after whole
update rounds rtol 1e-3 / atol 5e-5, clipped mean 4e-6 * max|v|."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from golden_util import load, agent_weights, pretrained    # noqa: E402
from oracle import rpbcac_oracle as O                        # noqa: E402  (checker only)

IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def close_w(got, want, rtol=1e-3, atol=5e-5):
    for n in range(len(want)):
        for k in range(6):
            np.testing.assert_allclose(np.asarray(got[n][k], np.float64), np.asarray(want[n][k], np.float64),
                                       rtol=rtol, atol=atol, err_msg=f"net {n} array {k}")


def synth(rs, B, NA=5, nrow=5):
    pos = rs.randint(0, nrow, size=(B, NA, 2))
    npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape), 0, nrow - 1)
    mean, std = (nrow - 1) / 2.0, np.std(np.arange(nrow))
    s = ((pos - mean) / std).astype(np.float32)
    ns = ((npos - mean) / std).astype(np.float32)
    a = rs.randint(0, 5, size=(B, NA, 1)).astype(np.float32)
    r = (-rs.randint(0, 2 * nrow, size=(B, NA, 1)) / 5.0).astype(np.float32)
    return s, ns, a, r


# ------------------------------------------------------------------------------------------ (a)
ONE_MALICIOUS = ['Cooperative'] * 4 + ['Malicious']
MIXED = ['Cooperative', 'Malicious', 'Greedy', 'Cooperative', 'Malicious']


@pytest.mark.parametrize("N,labels", [pytest.param(64, ONE_MALICIOUS, id="64"), pytest.param(128, ONE_MALICIOUS, id="128"),
                                      pytest.param(4096, ONE_MALICIOUS, id="4096"),
                                      pytest.param(1024, MIXED, id="1024-mixed")])
def test_malicious_round_at_staged_gather_shapes_matches_oracle(N, labels):
    need_gpu()
    from rcmarl.trainer import Trainer
    rs = np.random.RandomState(N)
    T1, gamma = 40, 0.9                          # 40 time rows: mini-batches of 32 and 8 time rows x N environments
    w, desired, _ = pretrained()
    agents = []
    for i, l in enumerate(labels):
        if l == 'Malicious':
            agents.append(O.MaliciousOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma,
                                                 critic_local_w=w[i][3] if len(w[i]) > 3 else None, dtype=np.float64))
        elif l == 'Greedy':
            agents.append(O.GreedyOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, dtype=np.float64))
        else:
            agents.append(O.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, H=1, dtype=np.float64))
    rs_perm = np.random.RandomState(N + 1)
    used = []

    def perm_rec(T):
        p = rs_perm.permutation(T)
        used.append(p)
        return p
    s, ns, a, r = synth(rs, T1 * N)
    want_loss = O.update_round(agents, labels, IN_NODES, s, ns, a, r, n_envs=N, n_epochs=2, n_actor_steps=T1,
                               common_reward=False, perm_source=perm_rec)
    it = iter(list(used))
    tr = Trainer(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
                 slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=64, perm_source=lambda T: next(it))
    tr.load_rows(s, ns, a, r)
    got_loss = tr.update_round()
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got_loss[k], want_loss[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        close_w(tr.get_weights(i), agents[i].get_parameters())


# ------------------------------------------------------------------------------------------ (b)
def _np_sums_chunked(w, x_of, y, B, chunk=1 << 19):
    """fp64 sum_rows e * dout/dtheta and sum e^2 over B rows, `chunk` rows at a time (x_of(lo, hi) -> (n, d) float64)."""
    w64 = O.cast_weights(w, np.float64)
    g_tot, l_tot = None, 0.0
    for lo in range(0, B, chunk):
        hi = min(B, lo + chunk)
        out, cch = O.mlp_forward(w64, x_of(lo, hi), cache=True)
        e = out - y[lo:hi].astype(np.float64).reshape(-1, 1)
        g = np.concatenate([t.reshape(-1) for t in O.mlp_backward(w64, cch, e)])
        g_tot = g if g_tot is None else g_tot + g
        l_tot += float((e * e).sum())
    return g_tot, l_tot


def test_c2_full_block_gradient_sums_match_numpy_fp64():
    need_gpu()
    from rcmarl import ops, nets, _lib as L
    NA, N, T = 5, 4096, 1000
    B = N * T                                                       # 4.096 M rows = one C2 block
    rs = np.random.RandomState(2)
    pos = rs.randint(0, 5, size=(B, NA, 2)).astype(np.int8)
    act = rs.randint(0, 5, size=(B, NA, 1)).astype(np.int8)
    npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape).astype(np.int8), 0, 4)
    std = np.float32(np.std(np.arange(5)))
    s = (pos.astype(np.float32) - 2.0) / std
    ns = (npos.astype(np.float32) - 2.0) / std
    sa = np.concatenate([s, act.astype(np.float32)], -1).reshape(B, 15)
    s2, ns2 = s.reshape(B, 10), ns.reshape(B, 10)
    tgt = (-rs.randint(0, 9, size=B) / 5.0).astype(np.float32) + 0.1 * rs.randn(B).astype(np.float32)
    w, _, _ = pretrained()
    wc, wt = w[0][1], w[0][2]
    dsa, dns, dt_ = (torch.as_tensor(x).cuda() for x in (sa, ns2, tgt))
    dr = torch.zeros(B, NA, device="cuda")
    dwc, dwt = torch.as_tensor(nets.pack(wc)).cuda(), torch.as_tensor(nets.pack(wt)).cuda()
    sc, st, sn = torch.zeros(662, device="cuda"), torch.zeros(762, device="cuda"), torch.zeros(662, device="cuda")
    rows = ops.make_rows(dsa, dns, dr, NA)
    ops.grad(rows, [ops.grad_job(dwc, dt_, sc, L.IN_S), ops.grad_job(dwt, dt_, st, L.IN_SA), ops.grad_job(dwc, dt_, sn, L.IN_NS)],
             L.LOSS_MSE)
    for got, wn, x in ((sc, wc, s2), (st, wt, sa), (sn, wc, ns2)):
        g, l = _np_sums_chunked(wn, lambda lo, hi, x=x: x[lo:hi].astype(np.float64), tgt, B)
        got = got.cpu().numpy().astype(np.float64)
        # fp32 accumulation of B terms in a fixed tree (lane -> warp -> CTA -> reduce kernel): error floor ~ eps * sqrt(B) * |term|
        scale = max(1.0, np.abs(g).max())
        np.testing.assert_allclose(got[:-1], g, rtol=1e-4, atol=2e-6 * scale)
        np.testing.assert_allclose(got[-1], l, rtol=2e-5)


# ------------------------------------------------------------------------------------------ (c)
@pytest.mark.parametrize("H", [0, 1, 2, 4])
def test_c5_clip_mean_matches_oracle_at_full_size(H):
    need_gpu()
    from rcmarl import ops
    g = torch.Generator(device="cuda"); g.manual_seed(H)
    X = torch.randn(64, 1 << 20, device="cuda", generator=g)
    X[:, ::100] = torch.round(X[:, ::100])                      # ties on 1 % of the columns (SURVEY 8d)
    got = ops.clip_mean(X, H).cpu().numpy().astype(np.float64)
    want = O.resilient_aggregation(X.cpu().numpy().astype(np.float64), H)
    np.testing.assert_allclose(got, want, rtol=0, atol=4e-6 * float(X.abs().max()))


# ------------------------------------------------------------------------------------------ (d)
def test_greedy_faulty_common_reward_run_matches_reference_train_run():
    need_gpu()
    from rcmarl.trainer import Trainer
    z = load("ref_adversaries.npz")
    w, desired, _ = pretrained()
    labels = [str(x) for x in z["run/labels"]]
    perms = [z[f"run/perm{j}"] for j in range(int(z["run/n_perms"]))]
    it = iter(perms)

    def perm_source(T):
        p = next(it)
        assert len(p) == T
        return p
    tr = Trainer(labels=labels, in_nodes=IN_NODES, weights=[x[:3] for x in w], desired=desired, n_envs=1, gamma=0.9, H=1,
                 fast_lr=0.01, slow_lr=0.002, max_ep_len=10, n_ep_fixed=25, n_epochs=2, buffer_size=100000,
                 capacity_times=600, common_reward=True, perm_source=perm_source)
    for rnd in (0, 1):
        sl = slice(250 * rnd, 250 * (rnd + 1))
        tr.load_rows(z["run/s"][sl], z["run/ns"][sl], z["run/a"][sl], z["run/r"][sl])
        tr.update_round()
    assert next(it, None) is None
    final = agent_weights(z, "run/final")
    for i in range(5):
        close_w(tr.get_weights(i), final[i])
