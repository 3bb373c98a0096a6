"""GPU parity of the selectable resilient aggregation rules (rcmarl_agg_rule: clip / trim / wmsr, include/rcmarl.h)
against the float64 oracle (tests/agg_oracle.py): the hidden-layer consensus with the rules mixed in one launch, the
team kernel at neighbour counts on both sides of its MAXN switches in both modes (agg_out / agg_in), Byzantine heads
and messages, the per-agent API, whole update rounds with per-agent rules, and the refusals.

Tolerances as in test_kernel_shapes_gpu.py: aggregated estimates rtol 1e-5 / atol 3e-6, projection sums rtol 1e-4
with an atol floor growing with sqrt(B), weights after a consensus step rtol 1e-4 / atol 1e-6, weights after whole
update rounds rtol 1e-3 / atol 5e-5 (as test_trainer_gpu.py)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import agg_oracle as AO                                # noqa: E402
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, rand_net, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_S, IN_SA = 0, 1
RULES = ("clip", "trim", "wmsr")
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def d_in(NA, kind):
    return 3 * NA if kind == IN_SA else 2 * NA


def valid_H(rs, rule, n_in):
    return int(rs.randint(0, min(7, (n_in - 1) // 2 if rule == "trim" else n_in - 1) + 1))


def neighbours(rs, own, n_in, n_msgs):
    """own first, repeats allowed, and own repeated once more when n_in >= 3 (values equal to own: W-MSR keeps them)."""
    nodes = [own] + [int(v) for v in rs.randint(0, n_msgs, size=n_in - 1)]
    if n_in >= 3:
        nodes[int(rs.randint(1, n_in))] = own
    return nodes


# ---------------------------------------------------------------------------------------------------------- consensus
@pytest.mark.parametrize("NA", [5, 16])
def test_consensus_hidden_rules_mixed_in_one_launch(K, NA):
    """Critic and TR jobs, n_in 1..16 with repeated in_nodes, the three rules mixed; output layers bitwise unchanged."""
    rs = np.random.RandomState(1100 + NA)
    dims = {IN_S: 2 * NA, IN_SA: 3 * NA}
    n_ag = 16
    nets = {k: [rand_net(rs, dims[k], 1) for _ in range(n_ag)] for k in dims}
    msgs = {k: to_dev(K, np.stack([K.nets.pack(w) for w in nets[k]]))[0] for k in dims}
    own = {k: [rand_net(rs, dims[k], 1) for _ in range(n_ag)] for k in dims}
    dst = {k: to_dev(K, np.stack([K.nets.pack(w) for w in own[k]]))[0] for k in dims}
    before = {k: v.clone() for k, v in dst.items()}
    nh = {k: K.nets.n_hidden_params(dims[k]) for k in dims}
    jobs, cfg = [], []
    for i in range(n_ag):
        for k, n_in in ((IN_S, 1 + i), (IN_SA, 16 - (5 * i) % 16)):
            rule = RULES[(i + k) % 3]
            nodes = neighbours(rs, i, n_in, n_ag)
            H = valid_H(rs, rule, n_in)
            jobs.append(K.ops.consensus_job(dst[k][i], msgs[k], msgs[k].shape[1], nh[k], nodes, H, rule))
            cfg.append((k, i, nodes, H, rule))
    assert len(jobs) == 32 and {c[4] for c in cfg} == set(RULES)
    K.ops.consensus_hidden(jobs)
    for k, i, nodes, H, rule in cfg:
        ag = AO.RPBCACOracleAgent(rand_net(rs, 2 * NA, 5), own[IN_S][i], own[IN_SA][i], 0.002, 0.01, H=H, dtype=f64,
                                  aggregation=rule)
        if k == IN_S:
            ag.resilient_consensus_critic_hidden([nets[k][m] for m in nodes])
            want = ag.critic
        else:
            ag.resilient_consensus_TR_hidden([nets[k][m] for m in nodes])
            want = ag.TR
        close(dst[k][i], K.nets.pack(want), rtol=1e-4, atol=1e-6, err_msg=f"kind {k} agent {i} n_in {len(nodes)} H {H} {rule}")
        assert torch.equal(dst[k][i][nh[k]:], before[k][i][nh[k]:])


def test_consensus_hidden_drops_byzantine_messages(K):
    """One neighbour sends 1e8, -1e8, +-inf, 1e30 in its hidden layers; with H = 1 every rule stays near the honest
    values (trim / wmsr drop it, clip clips it) and matches the oracle at absolute tolerance."""
    rs = np.random.RandomState(1200)
    NA, n_in = 5, 6
    din = 2 * NA
    honest = [rand_net(rs, din, 1) for _ in range(n_in)]
    bad = K.nets.pack(honest[3])
    nh = K.nets.n_hidden_params(din)
    bad[:nh] = np.resize(np.array([1e8, -1e8, np.inf, -np.inf, 1e30], np.float32), nh)
    stack = np.stack([K.nets.pack(w) for w in honest])
    stack[3] = bad
    bad_net = K.nets.unpack(bad, din, 1)
    dmsgs = to_dev(K, stack)[0]
    for rule in RULES:
        dst = to_dev(K, K.nets.pack(rand_net(rs, din, 1)))[0]
        K.ops.consensus_hidden([K.ops.consensus_job(dst, dmsgs, stack.shape[1], nh, list(range(n_in)), 1, rule)])
        ag = AO.RPBCACOracleAgent(rand_net(rs, din, 5), rand_net(rs, din, 1), rand_net(rs, 3 * NA, 1), 0.002, 0.01, H=1,
                                  dtype=f64, aggregation=rule)
        ag.resilient_consensus_critic_hidden([bad_net if m == 3 else honest[m] for m in range(n_in)])
        got = dst.cpu().numpy()[:nh]
        assert np.isfinite(got).all(), rule
        close(got, K.nets.pack(ag.critic)[:nh], rtol=0, atol=1e-5, err_msg=rule)


# ---------------------------------------------------------------------------------------------------------- team
def oracle_team(own, heads, X, H, rule):
    """fp64 aggregate of the neighbour-head estimates and the projection sums
    [sum c * phi (20) | sum c | sum (agg - pred) * c], c = (agg - pred) / (||phi||^2 + 1)."""
    w64 = O.cast_weights(own, f64)
    phi = O.mlp_features(w64, X.astype(f64))
    est = np.stack([(phi @ np.asarray(m[4], f64) + np.asarray(m[5], f64))[:, 0] for m in heads])
    agg = AO.resilient_aggregation(est, H, rule)
    err = agg - (phi @ w64[4] + w64[5])[:, 0]
    c = err / ((phi * phi).sum(1) + 1.0)
    return agg, np.concatenate([phi.T @ c, [c.sum(), (err * c).sum()]])


def check_sums(got, want, B, msg):
    scale = max(1.0, np.abs(want[:21]).max())
    close(got, want, rtol=1e-4, atol=2e-6 * scale * B ** 0.5, err_msg=msg)


@pytest.mark.parametrize("NA", [5, 16])
def test_team_rules_across_neighbour_bounds_both_modes(K, NA):
    """rcmarl_team per rule with n_in 4 | 5, 8 | 9 and 16 (the MAXN switches) for both input kinds: agg_out and the
    projection sums against the oracle; then the agg_in mode fed with the kernel's own aggregates reproduces the sums
    whatever rule and H the job carries (the rule is unused there)."""
    rs = np.random.RandomState(1300 + NA)
    B = 3001
    s, ns, a, r = synth(rs, B, NA, 5 if NA == 5 else 10)
    X = {IN_S: s.reshape(B, -1), IN_SA: np.concatenate([s, a], -1).reshape(B, -1)}
    dsa, dns, dr = to_dev(K, X[IN_SA], ns.reshape(B, -1), r[:, :, 0])
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    msgs = {k: [rand_net(rs, d_in(NA, k), 1) for _ in range(16)] for k in (IN_S, IN_SA)}
    dmsgs = {k: to_dev(K, np.stack([K.nets.pack(w) for w in ws]))[0] for k, ws in msgs.items()}
    jobs, data = [], []
    for kind in (IN_S, IN_SA):
        for n_in in (4, 5, 8, 9, 16):
            rule = RULES[(n_in + kind) % 3]
            H = valid_H(rs, rule, n_in)
            own_i = int(rs.randint(0, 16))
            nodes = neighbours(rs, own_i, n_in, 16)
            own = rand_net(rs, d_in(NA, kind), 1)
            dw = to_dev(K, K.nets.pack(own))[0]
            sums = torch.full((22,), NAN, device=K.dev)
            agg = torch.full((B,), NAN, device=K.dev)
            P = K.L.param_count(d_in(NA, kind), 1)
            jobs.append(K.ops.team_job(dw, kind, dmsgs[kind], P, nodes, H, sums=sums, agg_out=agg, rule=rule))
            data.append(dict(kind=kind, n_in=n_in, H=H, rule=rule, own=own, dw=dw, heads=[msgs[kind][m] for m in nodes],
                             sums=sums, agg=agg))
    assert {d["rule"] for d in data} == set(RULES)
    K.ops.team(rows, jobs)
    for d in data:
        msg = f"kind {d['kind']} n_in {d['n_in']} H {d['H']} {d['rule']}"
        want_agg, want_sums = oracle_team(d["own"], d["heads"], X[d["kind"]], d["H"], d["rule"])
        close(d["agg"], want_agg, rtol=1e-5, atol=3e-6, err_msg="agg_out " + msg)
        check_sums(d["sums"], want_sums, B, "sums " + msg)
        d["want_sums"] = want_sums
    # agg_in mode: msgs / n_in / H / rule are not read, so even a rule that would be refused with msgs is accepted
    jobs_in = []
    for d in data:
        d["sums_in"] = torch.full((22,), NAN, device=K.dev)
        P = K.L.param_count(d_in(NA, d["kind"]), 1)
        jobs_in.append(K.ops.team_job(d["dw"], d["kind"], sums=d["sums_in"], agg_in=d["agg"], in_nodes=[0] * 4, H=3,
                                      rule="trim"))
    K.ops.team(rows, jobs_in)
    for d in data:
        check_sums(d["sums_in"], d["want_sums"], B, f"agg_in sums kind {d['kind']} n_in {d['n_in']}")
        close(d["sums_in"], d["sums"].cpu().numpy(), rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("bad_value", [1e8, np.inf, -np.inf])
def test_team_byzantine_head(K, bad_value):
    """One neighbour's head predicts bad_value for every row (W3 = 0, b3 = bad_value); with H = 1 the aggregate stays
    finite under every rule and matches the oracle at absolute tolerance."""
    rs = np.random.RandomState(1400)
    NA, B, n_in = 5, 2001, 5
    s, ns, a, r = synth(rs, B, NA)
    X = s.reshape(B, -1)
    dsa, dns, dr = to_dev(K, np.concatenate([s, a], -1).reshape(B, -1), ns.reshape(B, -1), r[:, :, 0])
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    heads = [rand_net(rs, 2 * NA, 1) for _ in range(n_in)]
    heads[2][4] = np.zeros_like(heads[2][4])
    heads[2][5] = np.full_like(heads[2][5], bad_value)
    dmsgs = to_dev(K, np.stack([K.nets.pack(w) for w in heads]))[0]
    for rule in RULES:
        own = rand_net(rs, 2 * NA, 1)
        dw = to_dev(K, K.nets.pack(own))[0]
        sums = torch.full((22,), NAN, device=K.dev)
        agg = torch.full((B,), NAN, device=K.dev)
        K.ops.team(rows, [K.ops.team_job(dw, IN_S, dmsgs, dmsgs.shape[1], list(range(n_in)), 1, sums=sums, agg_out=agg,
                                         rule=rule)])
        want_agg, want_sums = oracle_team(own, heads, X, 1, rule)
        assert torch.isfinite(agg).all() and torch.isfinite(sums).all(), rule
        close(agg, want_agg, rtol=0, atol=1e-5, err_msg=rule)
        check_sums(sums, want_sums, B, rule)


# ---------------------------------------------------------------------------------------------------------- agent API
def build_models(w_agent, NA=5):
    from tensorflow import keras

    def seq(f, n_out, act):
        return keras.Sequential([keras.Input(shape=(NA, f)), keras.layers.Flatten(),
                                 keras.layers.Dense(20, activation=keras.layers.LeakyReLU(alpha=0.1)),
                                 keras.layers.Dense(20, activation=keras.layers.LeakyReLU(alpha=0.1)),
                                 keras.layers.Dense(n_out, activation=act)])
    actor, critic, tr = seq(2, 5, 'softmax'), seq(2, 1, None), seq(3, 1, None)
    actor.set_weights(w_agent[0]); critic.set_weights(w_agent[1]); tr.set_weights(w_agent[2])
    return actor, critic, tr


@pytest.mark.parametrize("rule", ["trim", "wmsr"])
def test_rpbcac_agent_methods_with_a_rule(K, rule):
    """RPBCAC_agent(..., aggregation=rule): hidden consensus, estimate consensus, projection step and
    _resilient_aggregation against the oracle agent built with the same rule."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H = 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule)
    ora = AO.RPBCACOracleAgent(w[0][0], w[0][1], w[0][2], 0.002, 0.01, 0.9, H=H, dtype=f64, aggregation=rule)
    nbrs = [0, 1, 0, 2, 4]                                             # own repeated: ties with own
    cmsgs = [list(w[j][1]) for j in nbrs]
    tmsgs = [list(w[j][2]) for j in nbrs]
    ag.resilient_consensus_critic_hidden(cmsgs)
    ag.resilient_consensus_TR_hidden(tmsgs)
    ora.resilient_consensus_critic_hidden(cmsgs)
    ora.resilient_consensus_TR_hidden(tmsgs)
    for k in range(6):
        close(ag.critic.get_weights()[k], ora.critic[k], rtol=1e-4, atol=1e-6)
        close(ag.TR.get_weights()[k], ora.TR[k], rtol=1e-4, atol=1e-6)
    cagg, tagg = ag.resilient_consensus_critic(s, cmsgs), ag.resilient_consensus_TR(sa, tmsgs)
    wc, wt = ora.resilient_consensus_critic(s, cmsgs), ora.resilient_consensus_TR(sa, tmsgs)
    close(cagg.numpy(), wc, rtol=1e-5, atol=3e-6)
    close(tagg.numpy(), wt, rtol=1e-5, atol=3e-6)
    ag.critic_update_team(s, cagg)
    ag.TR_update_team(sa, tagg)
    ora.critic_update_team(s, wc)
    ora.TR_update_team(sa, wt)
    for k in range(6):
        close(ag.critic.get_weights()[k], ora.critic[k], rtol=1e-4, atol=1e-6)
        close(ag.TR.get_weights()[k], ora.TR[k], rtol=1e-4, atol=1e-6)
    rs = np.random.RandomState(1500)
    v = rs.randint(-3, 4, size=(7, 3, 11)).astype(np.float32)           # ties
    v[:, 0] = rs.randn(7, 11)
    v[3, 1] = np.inf
    for H_ in (0, 1, 3):
        ag.H = H_
        close(ag._resilient_aggregation(v).numpy(), AO.resilient_aggregation(v.astype(f64), H_, rule), rtol=1e-5, atol=1e-6)


def test_rpbcac_agent_explicit_clip_matches_the_golden_vectors(K):
    from agents.resilient_CAC_agents import RPBCAC_agent
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    for H in (0, 1):
        actor, critic, tr = build_models(w[0])
        ag = RPBCAC_agent(actor, critic, tr, slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation="clip")
        close(ag._resilient_aggregation(z[f"agg/n4_H{H}_in"]).numpy(), z[f"agg/n4_H{H}_out"], rtol=1e-6, atol=2e-6)


# ---------------------------------------------------------------------------------------------------------- update rounds
def make_agents(w, labels, rules, H, gamma):
    ags = []
    for i, l in enumerate(labels):
        if l == "Cooperative":
            ags.append(AO.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, H=H, dtype=f64,
                                            aggregation=rules[i]))
        else:
            ags.append(O.MaliciousOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, critic_local_w=w[i][3],
                                              dtype=f64))
    return ags


def close_w(got, want, rtol=1e-3, atol=5e-5, msg=""):
    for n in range(len(want)):
        for k in range(6):
            close(got[n][k], want[n][k], rtol=rtol, atol=atol, err_msg=f"{msg} net {n} array {k}")


@pytest.mark.parametrize("N", [1, 64])
def test_update_round_with_per_agent_rules(K, N):
    """Two update rounds, cooperative agents on trim / wmsr / clip / wmsr (H = 1 of 4 neighbours) plus a Malicious
    agent, against the oracle's update_round; then aggregation="clip" given explicitly is bitwise equal to omitting it."""
    from rcmarl.trainer import Trainer
    w, desired, labels = pretrained()
    assert labels == ["Cooperative"] * 4 + ["Malicious"]
    rules = ["trim", "wmsr", "clip", "wmsr", "clip"]
    gamma, T = 0.9, 40
    rs = np.random.RandomState(1600 + N)
    s, ns, a, r = synth(rs, T * N)
    agents = make_agents(w, labels, rules, 1, gamma)
    prs = np.random.RandomState(1700)
    used = []

    def rec(T_):
        p = prs.permutation(T_)
        used.append(p)
        return p
    want = AO.update_round(agents, labels, IN_NODES, s, ns, a, r, n_envs=N, n_epochs=2, n_actor_steps=T,
                           common_reward=False, perm_source=rec)
    cfg = dict(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000)
    it = iter(list(used))
    tr = Trainer(aggregation=rules, perm_source=lambda T_: next(it), **cfg)
    tr.load_rows(s, ns, a, r)
    got = tr.update_round()
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({rules[i]})")
    # the default is the reference's clipped mean, bit for bit
    outs = []
    for kw in ({}, {"aggregation": "clip"}, {"aggregation": ["clip"] * 5}):
        it = iter(list(used))
        t2 = Trainer(perm_source=lambda T_: next(it), **cfg, **kw)
        t2.load_rows(s, ns, a, r)
        t2.update_round()
        outs.append([t2.actor.clone(), t2.critic.clone(), t2.tr.clone(), t2.critic_local.clone()])
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(outs[0], o))
    assert not torch.equal(outs[0][1], tr.critic)                       # and the other rules do change the result


# ---------------------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_everything_untouched(K):
    """An unknown rule, or trim with 2H >= n_in, refuses the whole call before any launch: no destination, sum or
    aggregate is written, for the valid jobs of the same call either."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    rs = np.random.RandomState(1800)
    NA = 5
    stack = to_dev(K, np.stack([K.nets.pack(rand_net(rs, 2 * NA, 1)) for _ in range(6)]))[0]
    P = stack.shape[1]
    nh = K.nets.n_hidden_params(2 * NA)
    dst = to_dev(K, np.stack([K.nets.pack(rand_net(rs, 2 * NA, 1)) for _ in range(2)]))[0]
    before = dst.clone()
    ok = K.ops.consensus_job(dst[0], stack, P, nh, [0, 1, 2, 3], 1, "trim")
    for bad in (K.ops.consensus_job(dst[1], stack, P, nh, [0, 1, 2, 3], 2, "trim"),      # 2H >= n_in
                K.ops.consensus_job(dst[1], stack, P, nh, [0, 1, 2, 3], 1, 3),           # unknown rule id
                K.ops.consensus_job(dst[1], stack, P, nh, [0, 1, 2, 3], 1, -1)):
        with pytest.raises(K.L.RcmarlError):
            K.ops.consensus_hidden([ok, bad])
        torch.cuda.synchronize()
        assert torch.equal(dst, before)
    B = 500
    s, ns, a, r = synth(rs, B, NA)
    dsa, dns, dr = to_dev(K, np.concatenate([s, a], -1).reshape(B, -1), ns.reshape(B, -1), r[:, :, 0])
    rows = K.ops.make_rows(dsa, dns, dr, NA)
    sums = torch.full((2, 22), NAN, device=K.dev)
    agg = torch.full((2, B), NAN, device=K.dev)
    good = K.ops.team_job(dst[0], IN_S, stack, P, [0, 1, 2], 1, sums=sums[0], agg_out=agg[0], rule="wmsr")
    for bad in (K.ops.team_job(dst[1], IN_S, stack, P, [0, 1, 2, 3, 4, 5], 3, sums=sums[1], agg_out=agg[1], rule="trim"),
                K.ops.team_job(dst[1], IN_S, stack, P, [0, 1, 2], 1, sums=sums[1], agg_out=agg[1], rule=7)):
        with pytest.raises(K.L.RcmarlError):
            K.ops.team(rows, [good, bad])
        torch.cuda.synchronize()
        assert torch.isnan(sums).all() and torch.isnan(agg).all()
    # the per-agent API: the library's refusal reaches the caller and the agent's networks stay as they were
    w, _, _ = pretrained()
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=2, aggregation="trim")
    wc, wt = ag.critic.get_weights(), ag.TR.get_weights()
    msgs = [list(w[j][1]) for j in (0, 1, 2, 4)]
    with pytest.raises(K.L.RcmarlError):
        ag.resilient_consensus_critic_hidden(msgs)
    with pytest.raises(K.L.RcmarlError):
        ag.resilient_consensus_critic(s, msgs)
    with pytest.raises(K.L.RcmarlError):
        ag._resilient_aggregation(np.zeros((4, 3), np.float32))
    for k in range(6):
        assert np.array_equal(ag.critic.get_weights()[k], wc[k]) and np.array_equal(ag.TR.get_weights()[k], wt[k])
    with pytest.raises(K.L.RcmarlError):
        RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=1, aggregation="median")
