"""GPU parity: every C-ABI entry point (include/rcmarl.h) against the CPU oracle
(oracle/rpbcac_oracle.py, float64 mode as the yardstick) on the same seeded inputs.

Tolerances (SURVEY 8d): forward outputs rtol 1e-5 / atol 2e-6; gradients / weights after
a fit or projection step rtol 1e-4 / atol 1e-6 (the reduction order over rows differs);
aggregation atol 4e-6 * max|v|; discrete outputs (actions, positions, rewards) exact.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from golden_util import pretrained                     # noqa: E402
from kernel_util import close, load_kernels, rand_net, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,H,P", [(4, 0, 661), (4, 1, 640), (6, 2, 1421), (9, 4, 4096), (3, 1, 37),
                                    (16, 7, 1000), (64, 4, 65536), (64, 1, 65537), (5, 2, 8), (1, 0, 16), (8, 3, 4096),
                                    (17, 5, 2048), (24, 6, 1024), (64, 2, 4100)])
def test_clip_mean_matches_oracle(K, n, H, P):
    rs = np.random.RandomState(n * 131 + H)
    v = rs.randn(n, P).astype(np.float32)
    v[:, ::7] = np.round(v[:, ::7])                       # ties
    v[:, 1::11] = v[0:1, 1::11]                           # everybody equal to own
    want = O.resilient_aggregation(v.astype(np.float64), H)
    got = K.ops.clip_mean(to_dev(K, v)[0], H)
    close(got, want, rtol=0, atol=4e-6 * np.abs(v).max())
    if H == 0:                                            # plain mean
        close(got, v.astype(np.float64).mean(0), rtol=0, atol=4e-6 * np.abs(v).max())


@pytest.mark.parametrize("n,H,P", [(4, 1, 640), (6, 2, 1421), (64, 4, 4096), (64, 1, 4099), (4, 0, 64)])
def test_clip_mean_is_robust_to_adversarial_outliers(K, n, H, P):
    """One Byzantine neighbour sends 1e8 / -3e30 / +-inf: tf.clip_by_value clips first and averages afterwards
    (agents/resilient_CAC_agents.py:55-56), so with H >= 1 the result stays at the honest values.  ABSOLUTE tolerance
    (not scaled by max|v|): a single-pass sum that contains the outlier would lose the honest values entirely."""
    rs = np.random.RandomState(n + H)
    v = (0.1 + 0.01 * rs.randn(n, P)).astype(np.float32)
    bad = [1e8, -3e30, np.inf, -np.inf]
    for j in range(P):
        if j % 3 == 0 and n > 1:
            v[1 + (j % (n - 1)), j] = bad[(j // 3) % 4]      # never the own row
    want = O.resilient_aggregation(v.astype(np.float64), H)
    got = K.ops.clip_mean(to_dev(K, v)[0], H).cpu().numpy().astype(np.float64)
    if H >= 1:
        assert np.isfinite(want).all() and np.abs(want - 0.1).max() < 0.1
        np.testing.assert_allclose(got, want, rtol=0, atol=2e-6)
    else:                                                        # H = 0 is the plain mean: outliers pass through
        fin = np.isfinite(want)
        np.testing.assert_allclose(got[fin], want[fin], rtol=1e-5, atol=2e-6)
        assert np.array_equal(np.isinf(got[~fin]) | np.isnan(got[~fin]), np.ones((~fin).sum(), bool))


def test_clip_mean_rejects_bad_args(K):
    v = torch.zeros(4, 8, device=K.dev)
    with pytest.raises(K.L.RcmarlError):
        K.ops.clip_mean(v, 4)                             # H >= n
    assert K.ops.clip_mean(torch.zeros(4, 0, device=K.dev), 1).numel() == 0   # empty input


def test_clip_mean_strided_rows_and_idempotence(K):
    rs = np.random.RandomState(0)
    big = to_dev(K, rs.randn(6, 1024).astype(np.float32))[0]
    view = big[:, :512]                                   # row stride 1024
    want = O.resilient_aggregation(view.cpu().numpy().astype(np.float64), 2)
    close(K.ops.clip_mean(view, 2), want, rtol=0, atol=2e-5)
    same = big[:1].repeat(6, 1).contiguous()
    close(K.ops.clip_mean(same, 2), same[0].cpu().numpy(), rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NA,nrow", [(5, 5), (16, 10)])
def test_values_td_target_and_td_error(K, NA, nrow):
    rs = np.random.RandomState(1)
    B = 777
    s, ns, a, r = synth(rs, B, NA, nrow)
    sa = np.concatenate([s, a], -1)
    wc, wt = rand_net(rs, 2 * NA, 1), rand_net(rs, 3 * NA, 1)
    dsa, dns, dr = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1))
    dwc, dwt = to_dev(K, K.nets.pack(wc), K.nets.pack(wt))
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    out1 = torch.zeros(B, device=K.dev)
    out2 = torch.zeros(B, device=K.dev)
    gamma = 0.9
    K.ops.values(rows, [
        K.ops.value_job(out1, [(dwc, K.L.IN_NS, gamma)], add=dr, add_stride=NA, add_off=2, add_scale=1.0),
        K.ops.value_job(out2, [(dwt, K.L.IN_SA, 1.0), (dwc, K.L.IN_NS, gamma), (dwc, K.L.IN_S, -1.0)])])
    f64 = np.float64
    wc64, wt64 = O.cast_weights(wc, f64), O.cast_weights(wt, f64)
    V = O.mlp_forward(wc64, O.flatten_rows(s, f64))
    nV = O.mlp_forward(wc64, O.flatten_rows(ns, f64))
    TR = O.mlp_forward(wt64, O.flatten_rows(sa, f64))
    close(out1, (r[:, 2].astype(f64) + gamma * nV)[:, 0], rtol=1e-5, atol=3e-6)
    close(out2, (TR + gamma * nV - V)[:, 0], rtol=1e-5, atol=5e-6)


def test_values_actor_probs(K):
    rs = np.random.RandomState(2)
    NA, B = 5, 300
    s, ns, a, r = synth(rs, B)
    wa = rand_net(rs, 10, 5)
    dns = to_dev(K, s.reshape(B, -1))[0]
    dwa = to_dev(K, K.nets.pack(wa))[0]
    out = torch.zeros(B, 5, device=K.dev)
    rows = K.ops.make_rows(None, dns, None, NA)
    K.ops.values(rows, [K.ops.value_job(out, [(dwa, K.L.IN_NS, 1.0)], n_out=5, softmax=1)])
    want = O.softmax(O.mlp_forward(O.cast_weights(wa, np.float64), O.flatten_rows(s, np.float64)))
    close(out, want, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------
def oracle_mse_sums(w, x, y):
    """unscaled sums the kernel returns: d/dtheta of 0.5*sum(e^2) ... i.e. sum_rows e * dout/dtheta, and sum e^2."""
    f64 = np.float64
    w64 = O.cast_weights(w, f64)
    out, cch = O.mlp_forward(w64, x.astype(f64), cache=True)
    e = out - y.astype(f64).reshape(-1, 1)
    g = O.mlp_backward(w64, cch, e)
    return np.concatenate([a.reshape(-1) for a in g]), float((e * e).sum())


@pytest.mark.parametrize("NA,nrow,B", [(5, 5, 1), (5, 5, 31), (5, 5, 1000), (5, 5, 20000), (16, 10, 3000)])
def test_grad_mse_matches_oracle(K, NA, nrow, B):
    rs = np.random.RandomState(B + NA)
    s, ns, a, r = synth(rs, B, NA, nrow)
    sa = np.concatenate([s, a], -1)
    wc, wt = rand_net(rs, 2 * NA, 1), rand_net(rs, 3 * NA, 1)
    tgt_c, tgt_t = rs.randn(B).astype(np.float32), rs.randn(B).astype(np.float32)
    dsa, dns, dr, dtc, dtt = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1), tgt_c, tgt_t)
    dwc, dwt = to_dev(K, K.nets.pack(wc), K.nets.pack(wt))
    PC, PT = K.L.param_count(2 * NA, 1), K.L.param_count(3 * NA, 1)
    sc, st, sn = (torch.zeros(PC + 1, device=K.dev), torch.zeros(PT + 1, device=K.dev), torch.zeros(PC + 1, device=K.dev))
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    K.ops.grad(rows, [K.ops.grad_job(dwc, dtc, sc, K.L.IN_S), K.ops.grad_job(dwt, dtt, st, K.L.IN_SA),
                      K.ops.grad_job(dwc, dtt, sn, K.L.IN_NS)], K.L.LOSS_MSE)
    for got, w, x, y in ((sc, wc, s, tgt_c), (st, wt, sa, tgt_t), (sn, wc, ns, tgt_t)):
        g, l = oracle_mse_sums(w, O.flatten_rows(x, np.float64), y)
        scale = max(1.0, np.abs(g).max())
        close(got[:-1], g, rtol=1e-4, atol=2e-6 * scale * max(1, B) ** 0.5)
        close(got[-1], l, rtol=1e-5, atol=1e-6)


def test_grad_is_deterministic_and_handles_empty(K):
    rs = np.random.RandomState(5)
    NA, B = 5, 5000
    s, ns, a, r = synth(rs, B)
    sa = np.concatenate([s, a], -1)
    dsa, dns, dr, dt = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1), rs.randn(B).astype(np.float32))
    dw = to_dev(K, K.nets.pack(rand_net(rs, 10, 1)))[0]
    s1, s2 = torch.zeros(662, device=K.dev), torch.zeros(662, device=K.dev)
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    K.ops.grad(rows, [K.ops.grad_job(dw, dt, s1, K.L.IN_S)], K.L.LOSS_MSE)
    K.ops.grad(rows, [K.ops.grad_job(dw, dt, s2, K.L.IN_S)], K.L.LOSS_MSE)
    assert torch.equal(s1, s2)                            # fixed-order reductions: bitwise reproducible
    rows0 = K.ops.make_rows(dsa, dns, dr, NA, n_rows=0)
    s1.fill_(7.0)
    K.ops.grad(rows0, [K.ops.grad_job(dw, dt, s1, K.L.IN_S)], K.L.LOSS_MSE)
    assert float(s1.abs().max()) == 0.0                   # empty row set -> zero sums


def test_grad_minibatch_time_index_equals_gathered_rows(K):
    """Appendix C mini-batch: 32 time rows x all envs, addressed through time_idx."""
    rs = np.random.RandomState(6)
    NA, N, T = 5, 24, 40
    B = N * T
    s, ns, a, r = synth(rs, B)
    sa = np.concatenate([s, a], -1)
    w = rand_net(rs, 15, 1)
    tgt = rs.randn(B).astype(np.float32)
    tidx = rs.permutation(T)[:32].astype(np.int32)
    dsa, dns, dr, dt, dti = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1), tgt, tidx)
    dw = to_dev(K, K.nets.pack(w))[0]
    sums = torch.zeros(762, device=K.dev)
    rows = K.ops.make_rows(dsa, dns, dr, NA, time_idx=dti, n_envs=N)
    K.ops.grad(rows, [K.ops.grad_job(dw, dt, sums, K.L.IN_SA)], K.L.LOSS_MSE)
    idx = O.expand_time_perm(tidx, N)
    g, l = oracle_mse_sums(w, O.flatten_rows(sa[idx], np.float64), tgt[idx])
    close(sums[:-1], g, rtol=1e-4, atol=1e-4)
    close(sums[-1], l, rtol=1e-5)


@pytest.mark.parametrize("NA,nrow", [(5, 5), (16, 10)])
def test_local_fit_five_steps_matches_oracle(K, NA, nrow):
    """critic_update_local / TR_update_local (agents/resilient_CAC_agents.py:103-140): TD target from the
    pre-fit weights, 5 full-batch SGD steps; message copy, own weights untouched."""
    rs = np.random.RandomState(7)
    B, lr, gamma = 1200, 0.01, 0.9
    s, ns, a, r = synth(rs, B, NA, nrow)
    sa = np.concatenate([s, a], -1)
    wc, wt = rand_net(rs, 2 * NA, 1), rand_net(rs, 3 * NA, 1)
    dsa, dns, dr = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1))
    dwc, dwt = to_dev(K, K.nets.pack(wc), K.nets.pack(wt))
    PC, PT = K.L.param_count(2 * NA, 1), K.L.param_count(3 * NA, 1)
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    tgt_c = torch.zeros(B, device=K.dev)
    tgt_t = dr[:, 1].contiguous()
    K.ops.values(rows, [K.ops.value_job(tgt_c, [(dwc, K.L.IN_NS, gamma)], add=dr, add_stride=NA, add_off=1)])
    msg_c, msg_t = torch.zeros(PC, device=K.dev), torch.zeros(PT, device=K.dev)
    sc, st = torch.zeros(PC + 1, device=K.dev), torch.zeros(PT + 1, device=K.dev)
    loss = torch.zeros(2, device=K.dev)
    for step in range(5):
        src_c, src_t = (dwc, dwt) if step == 0 else (msg_c, msg_t)
        K.ops.grad(rows, [K.ops.grad_job(src_c, tgt_c, sc, K.L.IN_S), K.ops.grad_job(src_t, tgt_t, st, K.L.IN_SA)],
                   K.L.LOSS_MSE)
        K.ops.sgd_apply([K.ops.sgd_job(msg_c, src_c, sc, PC, lr * 2.0 / B, loss_out=loss[0:1] if step == 0 else None,
                                       loss_coef=1.0 / B),
                         K.ops.sgd_job(msg_t, src_t, st, PT, lr * 2.0 / B, loss_out=loss[1:2] if step == 0 else None,
                                       loss_coef=1.0 / B)])
    ag = O.RPBCACOracleAgent(rand_net(rs, 2 * NA, 5), wc, wt, 0.002, lr, gamma, dtype=np.float64)
    wc_new, lc = ag.critic_update_local(s, ns, r[:, 1])
    wt_new, lt = ag.TR_update_local(sa, r[:, 1])
    close(msg_c, K.nets.pack(wc_new), rtol=1e-4, atol=1e-6)
    close(msg_t, K.nets.pack(wt_new), rtol=1e-4, atol=1e-6)
    close(loss, [lc, lt], rtol=1e-5)
    close(dwc, K.nets.pack(wc), rtol=0, atol=0)              # own weights untouched


@pytest.mark.parametrize("NA,nrow", [(5, 5), (16, 10)])
def test_actor_ce_grad_and_keras_adam(K, NA, nrow):
    rs = np.random.RandomState(8)
    B, lr = 900, 0.002
    s, ns, a, r = synth(rs, B, NA, nrow)
    sa = np.concatenate([s, a], -1)
    wa = rand_net(rs, 2 * NA, 5)
    delta = rs.randn(B).astype(np.float32)
    agent = 3
    PA = K.L.param_count(2 * NA, 5)
    dsa, dns, dr, dd = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1), delta)
    theta = to_dev(K, K.nets.pack(wa))[0]
    m, v, sums, loss = (torch.zeros(PA, device=K.dev), torch.zeros(PA, device=K.dev), torch.zeros(PA + 1, device=K.dev),
                        torch.zeros(1, device=K.dev))
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    adam = O.KerasAdam(lr)
    w64 = O.cast_weights(wa, np.float64)
    for t in range(1, 4):
        K.ops.grad(rows, [K.ops.grad_job(theta, dd, sums, K.L.IN_S, action_agent=agent)], K.L.LOSS_CE)
        K.ops.adam_apply([K.ops.adam_job(theta, m, v, sums, PA, 1.0 / B, K.ops.keras_adam_lr_t(lr, t), loss_out=loss,
                                         loss_coef=1.0 / B)])
        w64, l64 = O.actor_ce_step(w64, adam, O.flatten_rows(s, np.float64), a[:, agent], delta.astype(np.float64))
        close(loss, [l64], rtol=1e-4, atol=1e-6)
        close(theta, K.nets.pack(w64), rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize("NA,nrow,n_in,H", [(5, 5, 4, 0), (5, 5, 4, 1), (16, 10, 6, 2), (5, 5, 1, 0), (16, 10, 16, 7),
                                            (16, 10, 9, 4), (5, 5, 5, 2)])
def test_team_estimates_and_projection(K, NA, nrow, n_in, H):
    rs = np.random.RandomState(9 + H)
    B, lr = 1500, 0.01
    s, ns, a, r = synth(rs, B, NA, nrow)
    sa = np.concatenate([s, a], -1)
    n_ag = max(NA, n_in)
    nets_c = [rand_net(rs, 2 * NA, 1) for _ in range(n_ag)]
    nets_t = [rand_net(rs, 3 * NA, 1) for _ in range(n_ag)]
    own_c, own_t = rand_net(rs, 2 * NA, 1), rand_net(rs, 3 * NA, 1)
    in_nodes = list(rs.permutation(n_ag)[:n_in])
    PC, PT = K.L.param_count(2 * NA, 1), K.L.param_count(3 * NA, 1)
    dsa, dns, dr = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1))
    msgs_c = to_dev(K, np.stack([K.nets.pack(w) for w in nets_c]))[0]
    msgs_t = to_dev(K, np.stack([K.nets.pack(w) for w in nets_t]))[0]
    dwc, dwt = to_dev(K, K.nets.pack(own_c), K.nets.pack(own_t))
    sums = torch.zeros(2, 22, device=K.dev)
    agg = torch.zeros(2, B, device=K.dev)
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    K.ops.team(rows, [K.ops.team_job(dwc, K.L.IN_S, msgs_c, PC, in_nodes, H, sums=sums[0], agg_out=agg[0]),
                      K.ops.team_job(dwt, K.L.IN_SA, msgs_t, PT, in_nodes, H, sums=sums[1], agg_out=agg[1])])
    new_c, new_t = dwc.clone(), dwt.clone()
    K.ops.sgd_apply([K.ops.sgd_job(new_c, dwc, sums[0], PC, -1.0 / B, first=PC - 21),
                     K.ops.sgd_job(new_t, dwt, sums[1], PT, -1.0 / B, first=PT - 21)])
    ag = O.RPBCACOracleAgent(rand_net(rs, 2 * NA, 5), own_c, own_t, 0.002, lr, 0.9, H=H, dtype=np.float64)
    cm, tm = [nets_c[i] for i in in_nodes], [nets_t[i] for i in in_nodes]
    cagg = ag.resilient_consensus_critic(s, cm)
    tagg = ag.resilient_consensus_TR(sa, tm)
    close(agg[0], cagg[:, 0], rtol=1e-5, atol=5e-6)
    close(agg[1], tagg[:, 0], rtol=1e-5, atol=5e-6)
    ag.critic_update_team(s, cagg)
    ag.TR_update_team(sa, tagg)
    close(new_c, K.nets.pack(ag.critic), rtol=1e-4, atol=2e-6)
    close(new_t, K.nets.pack(ag.TR), rtol=1e-4, atol=2e-6)
    # two-call form of the reference API: estimates first, projection from a supplied agg
    sums2 = torch.zeros(22, device=K.dev)
    K.ops.team(rows, [K.ops.team_job(dwc, K.L.IN_S, sums=sums2, agg_in=agg[0])])
    close(sums2[:21], sums[0][:21].cpu().numpy(), rtol=1e-6, atol=1e-7)


def test_consensus_hidden_matches_oracle(K):
    rs = np.random.RandomState(10)
    NA = 5
    nets_c = [rand_net(rs, 10, 1) for _ in range(NA)]
    PC = K.L.param_count(10, 1)
    msgs = to_dev(K, np.stack([K.nets.pack(w) for w in nets_c]))[0]
    in_nodes = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1]]
    own = to_dev(K, np.stack([K.nets.pack(rand_net(rs, 10, 1)) for _ in range(4)]))[0]
    before = own.clone()
    nh = K.nets.n_hidden_params(10)
    K.ops.consensus_hidden([K.ops.consensus_job(own[i], msgs, PC, nh, in_nodes[i], 1) for i in range(4)])
    for i in range(4):
        ag = O.RPBCACOracleAgent(nets_c[0], K.nets.unpack(before[i].cpu().numpy(), 10, 1), nets_c[0], 0.002, 0.01,
                                 H=1, dtype=np.float64)
        ag.resilient_consensus_critic_hidden([nets_c[j] for j in in_nodes[i]])
        close(own[i], K.nets.pack(ag.critic), rtol=1e-6, atol=1e-6)
        assert torch.equal(own[i][nh:], before[i][nh:])      # output layer untouched (:153)


def test_reward_mix_matches_reference_order(K):
    rs = np.random.RandomState(11)
    r = (-rs.randint(0, 9, size=(1000, 5)) / 5.0).astype(np.float32)
    got = K.ops.reward_mix(to_dev(K, r)[0], [0, 1, 2, 3])
    want = np.zeros(1000, np.float32)
    for i in range(4):
        want = want + r[:, i] / np.float32(4)
    assert np.array_equal(got.cpu().numpy(), want)


# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NA,nrow,N", [(5, 5, 1), (5, 5, 64), (16, 10, 8)])
def test_rollout_matches_oracle_with_injected_randomness(K, NA, nrow, N):
    rs = np.random.RandomState(12 + N)
    n_ep, L_, gamma = 6, 20, 0.9
    labels = ['Cooperative'] * NA
    if NA == 5:
        w, desired, _ = pretrained()
        actors, critics = [w[i][0] for i in range(5)], [w[i][1] for i in range(5)]
    else:
        actors = [rand_net(rs, 2 * NA, 5) for _ in range(NA)]
        critics = [rand_net(rs, 2 * NA, 1) for _ in range(NA)]
        desired = rs.randint(0, nrow, size=(NA, 2))
    init = rs.randint(0, nrow, size=(n_ep, N, NA, 2)).astype(np.int32)
    init[0, 0] = desired                                   # start on the goal: reward-0 branch
    U = rs.rand(n_ep, L_, N, NA, 3).astype(np.float32)
    agents = [O.RPBCACOracleAgent(actors[i], critics[i], rand_net(rs, 3 * NA, 1), 0.002, 0.01, gamma) for i in range(NA)]
    env = O.GridWorldOracle(nrow, nrow, NA, desired, n_envs=N)
    S, NS_, A, R, est, ret = O.rollout_block(env, agents, labels, n_episodes=n_ep, max_ep_len=L_, gamma=gamma,
                                             init_states=init, uniforms=U)
    T = n_ep * L_
    dsa = torch.zeros(T * N, 3 * NA, device=K.dev)
    dns = torch.zeros(T * N, 2 * NA, device=K.dev)
    dr = torch.zeros(T * N, NA, device=K.dev)
    dest = torch.zeros(n_ep, N, NA, device=K.dev)
    dret = torch.zeros(n_ep, N, NA, device=K.dev)
    aw, cw, ddes, dinit, dU = to_dev(K, np.stack([K.nets.pack(x) for x in actors]),
                                     np.stack([K.nets.pack(x) for x in critics]),
                                     np.asarray(desired, np.int32), init, U)
    K.ops.rollout(aw, cw, ddes, dsa, dns, dr, 0, dest, dret, n_envs=N, n_agents=NA, n_episodes=n_ep, max_ep_len=L_,
                  nrow=nrow, ncol=nrow, gamma=gamma, mu=0.1, uniforms=dU, init_state=dinit)
    got_sa = dsa.cpu().numpy().reshape(T * N, NA, 3)
    want_s = S.astype(np.float32)
    # actions may differ only where a uniform sits within fp32 noise of a CDF edge; then the row diverges.
    act_equal = got_sa[:, :, 2] == A[:, :, 0]
    assert act_equal.mean() > 0.999, act_equal.mean()
    ok_ep = np.ones((n_ep, N), bool)                       # episodes free of any such tie
    bad = np.argwhere(~act_equal)
    for row, _ag in bad:
        t, e = divmod(row, N)
        ok_ep[t // L_, e] = False
    mask = np.repeat(ok_ep, L_, axis=0).reshape(-1)
    assert np.array_equal(got_sa[mask][:, :, :2], want_s[mask])
    assert np.array_equal(dns.cpu().numpy().reshape(T * N, NA, 2)[mask], NS_.astype(np.float32)[mask])
    assert np.array_equal(dr.cpu().numpy()[mask], R.astype(np.float32)[mask][:, :, 0])
    close(dest.cpu().numpy()[ok_ep], est[ok_ep], rtol=1e-5, atol=3e-6)
    close(dret.cpu().numpy()[ok_ep], ret[ok_ep], rtol=1e-5, atol=1e-5)


def test_rollout_philox_statistics_and_determinism(K):
    """Without injected randomness: same seed -> identical rows; env shards are independent of the launch
    decomposition (env_offset); resets are uniform over the grid; mu-mixture is respected."""
    NA, N, n_ep, L_ = 5, 256, 10, 20
    w, desired, _ = pretrained()
    aw, cw = to_dev(K, np.stack([K.nets.pack(w[i][0]) for i in range(5)]), np.stack([K.nets.pack(w[i][1]) for i in range(5)]))
    ddes = to_dev(K, np.asarray(desired, np.int32))[0]

    def run(n_envs, env_offset, seed):
        T = n_ep * L_
        sa = torch.zeros(T * n_envs, 15, device=K.dev)
        ns = torch.zeros(T * n_envs, 10, device=K.dev)
        r = torch.zeros(T * n_envs, 5, device=K.dev)
        est = torch.zeros(n_ep, n_envs, 5, device=K.dev)
        ret = torch.zeros(n_ep, n_envs, 5, device=K.dev)
        K.ops.rollout(aw, cw, ddes, sa, ns, r, 0, est, ret, n_envs=n_envs, n_agents=NA, n_episodes=n_ep,
                      max_ep_len=L_, nrow=5, ncol=5, gamma=0.9, seed=seed, env_offset=env_offset)
        return sa.view(T, n_envs, 15), r.view(T, n_envs, 5)
    full, rf = run(N, 0, 99)
    again, _ = run(N, 0, 99)
    assert torch.equal(full, again)
    half, rh = run(N // 2, N // 2, 99)                      # second shard of a 2-way split
    assert torch.equal(full[:, N // 2:], half) and torch.equal(rf[:, N // 2:], rh)
    other, _ = run(N, 0, 100)
    assert not torch.equal(full, other)
    tx, _ty = K.ops.state_tables(5, 5)
    first = full[::L_, :, 0].cpu().numpy()                  # x of agent 0 at reset
    counts = np.array([(np.isclose(first, v)).sum() for v in tx])
    assert counts.sum() == first.size and counts.min() > 0.12 * first.size
    acts = full[:, :, 2::3].cpu().numpy()
    assert set(np.unique(acts)) <= {0.0, 1.0, 2.0, 3.0, 4.0}
    rewards = rf.cpu().numpy()
    assert rewards.max() <= 0.0 and rewards.min() >= -(8 + 1) / 5.0 - 1e-6


def test_env_step_matches_reference_fixture(K):
    from golden_util import load
    z = load("ref_env.npz")
    for tag, nrow, na in (("5x5", 5, 5), ("10x10", 10, 16), ("3x3", 3, 3)):
        S = z[f"{tag}/state_int"]
        state = torch.as_tensor(S[0:1].astype(np.int32)).to(K.dev).contiguous()
        des = torch.as_tensor(z[f"{tag}/desired"].astype(np.int32)).to(K.dev)
        for t in range(z[f"{tag}/action"].shape[0]):
            act = torch.as_tensor(z[f"{tag}/action"][t:t + 1].astype(np.float32)).to(K.dev)
            rew = K.ops.env_step(state, act, des, nrow)
            assert np.array_equal(state.cpu().numpy()[0], S[t + 1])
            assert np.array_equal(rew.cpu().numpy()[0], z[f"{tag}/reward_scaled"][t].astype(np.float32))


# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NA,nrow,N,T", [(5, 5, 64, 40), (5, 5, 24, 37), (16, 10, 64, 33), (5, 5, 1, 96)])
def test_minibatch_fit_persistent_kernel_matches_oracle_and_step_loop(K, NA, nrow, N, T):
    """rcmarl_minibatch_fit (ONE persistent kernel: parameters resident in shared memory, cross-CTA reduction through
    {value, sequence} cells) against (a) the fp64 oracle's fit_minibatch with the same injected permutations
    (agents/adversarial_CAC_agents.py:133,150,163: fit(batch_size=32, epochs=E), Appendix C batching) and (b) the
    per-step loop ops.minibatch_steps (rcmarl_grad -> rcmarl_sgd_apply, the data-parallel NCCL path) at world 1;
    and bitwise reproducibility of two runs."""
    rs = np.random.RandomState(NA + N + T)
    E, mb, lr = 3, 32, 0.01
    B = N * T
    s, ns, a, r = synth(rs, B, NA, nrow)
    sa = np.concatenate([s, a], -1)
    kinds = [K.L.IN_S, K.L.IN_SA, K.L.IN_S]
    nets0 = [rand_net(rs, 3 * NA if k == K.L.IN_SA else 2 * NA, 1) for k in kinds]
    tgts = [rs.randn(B).astype(np.float32) for _ in kinds]
    perms = np.stack([np.stack([rs.permutation(T) for _ in range(E)]) for _ in kinds]).astype(np.int32)     # [C, E, T]
    dsa, dns, dr = to_dev(K, sa.reshape(B, -1), ns.reshape(B, -1), r.reshape(B, -1))
    dperm = to_dev(K, perms)[0]
    dt = to_dev(K, *tgts)

    def run(persistent):
        ws = [to_dev(K, K.nets.pack(w))[0] for w in nets0]
        loss = torch.zeros(len(kinds), device=K.dev)
        gj, aj = [], []
        for c, kind in enumerate(kinds):
            n = ws[c].numel()
            sums = torch.zeros(n + 1, device=K.dev)
            g = K.ops.grad_job(ws[c], dt[c], sums, kind, time_idx=dperm)
            g.time_idx = dperm.data_ptr() + 4 * c * E * T
            gj.append(g)
            aj.append(K.ops.sgd_job(ws[c], ws[c], sums, n, 0.0, loss_out=loss[c:c + 1], loss_coef=1.0 / B, loss_accumulate=1))
        rows = K.ops.make_rows(dsa, dns, dr, NA, 0, 0, dperm, N)
        if persistent:
            cells = K.ops.MinibatchCells(len(kinds), K.L.param_count(3 * NA, 1))
            K.ops.minibatch_fit(rows, gj, aj, E, T, mb, lr, cells)
            K.ops.minibatch_fit(rows, gj, aj, E, T, mb, 0.0 * lr + 1e-30, cells)     # second call on the same cells: a no-op step size
        else:
            K.ops.minibatch_steps(rows, gj, aj, E, T, mb, [lr] * len(kinds))
        torch.cuda.synchronize()
        return [w.cpu().numpy() for w in ws], loss.cpu().numpy()
    w_p, loss_p = run(True)
    w_p2, _ = run(True)
    w_c, loss_c = run(False)
    for c, kind in enumerate(kinds):
        assert np.array_equal(w_p[c], w_p2[c])                                 # fixed-order reductions
        x = O.flatten_rows(sa if kind == K.L.IN_SA else s, np.float64)
        rp = [O.expand_time_perm(perms[c, e], N) for e in range(E)]
        w64, l64 = O.fit_minibatch(O.cast_weights(nets0[c], np.float64), x, tgts[c].astype(np.float64).reshape(-1, 1), lr, E,
                                   mb * N, rp)
        want = K.nets.pack(w64)
        np.testing.assert_allclose(w_p[c], want, rtol=2e-4, atol=2e-6)
        np.testing.assert_allclose(w_p[c], w_c[c], rtol=1e-5, atol=1e-6)
        # the second (tiny step size) call accumulated its own epoch-0 loss on top: compare the first call's share only
        np.testing.assert_allclose(loss_c[c], l64, rtol=1e-4)
    assert np.all(loss_p > loss_c * 1.05)                                      # two calls accumulated two epoch-0 losses
