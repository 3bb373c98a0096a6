"""The Philox branch of rcmarl_rollout -- what bench.py, main.py and every Trainer without injected randomness train on
-- pinned by an exact restatement of its random streams (tests/rollout_oracle.py, from include/rcmarl.h):

  (a) a Philox-mode launch is bitwise equal to the injected-mode launch fed the restated draws, for 5- and 16-agent
      instantiations with fewer active agents, square / non-square / 1x1 / 32x32 grids, partial CTAs, env offsets
      across the 2^32 boundary, an episode word that wraps, time_begin > 0 and mu in {0, 0.1, 1};
  (b) the same launches against O.rollout_block in fp64;
  (c) the block bench.py rolls out first (C2, 4096 environments, 50 x 20 steps, seed 1234) against the oracle;
  (d) the Trainer's default loop (no injected draws, rows or shuffles) teacher-forced per round against the oracle:
      rollout rows and logged means, the whole update round with the Trainer's own shuffles, and the Phase-IV trim;
  (e) training.train_RPBCAC's logged sim_data against the reference's formulas on the oracle's rollouts.

Actions, positions and rewards are compared exactly.  Where an action uniform lies within fp32 noise of a CDF edge the
fp32 and fp64 policies may pick different actions; such episodes ('ties', < 0.1 % of actions) are excluded row-exactly,
as in test_kernels_gpu.py.  Tolerances are those of DESIGN.md section 2."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import rollout_oracle as R                            # noqa: E402
import team_util as T16                               # noqa: E402
from golden_util import pretrained                    # noqa: E402
from kernel_util import close, load_kernels, rand_net, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                 # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
C = "Cooperative"
SEED2 = 0x9E3779B97F4A7C15                            # both key words non-zero
N_EP, LEN = 3, 7


@pytest.fixture(scope="module")
def K():
    return load_kernels()


# --------------------------------------------------------------------------------------------------- shared checks
def rows_of(sa, ns, r, NA, nact, t0, t1, N):
    """Time rows [t0, t1) of device buffers as the oracle's (s, ns, a, r) for agents 0 .. nact-1."""
    sa = sa[t0 * N:t1 * N].view(-1, NA, 3)[:, :nact].cpu().numpy()
    return (sa[:, :, :2], ns[t0 * N:t1 * N].view(-1, NA, 2)[:, :nact].cpu().numpy(), sa[:, :, 2:],
            r[t0 * N:t1 * N].view(-1, NA, 1)[:, :nact].cpu().numpy())


# --------------------------------------------------------------------------------------------------- (a), (b) kernel
#        NA nact nrow ncol     N  env_offset   episode_offset time_begin mu  seed
CASES = [(5, 5, 5, 5, 1, 0, 0, 0, 0.1, 0),
         (5, 3, 4, 6, 127, 2 ** 32 - 5, 12345, 7, 0.0, SEED2),
         (5, 1, 6, 4, 128, 2 ** 32 + 7, 2 ** 32 - 2, 0, 1.0, SEED2),
         (5, 5, 32, 32, 4096, 2 ** 32 + 7, 2 ** 32 - 2, 5, 0.1, SEED2),
         (5, 3, 5, 5, 129, 2 ** 32 - 5, 12345, 11, 0.0, 0),
         (5, 1, 1, 1, 1, 0, 12345, 0, 0.1, 0),
         (16, 16, 32, 32, 129, 0, 12345, 3, 0.1, SEED2),
         (16, 7, 1, 1, 4096, 2 ** 32 - 5, 0, 0, 0.1, 0),
         (16, 7, 4, 6, 127, 0, 2 ** 32 - 2, 0, 1.0, 0),
         (16, 16, 6, 4, 128, 2 ** 32 + 7, 0, 2, 0.1, SEED2)]
IDS = [f"NA{c[0]}-act{c[1]}-{c[2]}x{c[3]}-N{c[4]}-env{c[5]}-ep{c[6]}-t{c[7]}-mu{c[8]}-s{c[9] != 0:d}" for c in CASES]


def setup_case(K, case):
    NA, nact, nrow, ncol, N, env_off, ep_off, tb, mu, seed = case
    rs = np.random.RandomState(sum(case[:5]) % 1000)
    actors = [rand_net(rs, 2 * nact, 5) for _ in range(nact)]
    critics = [rand_net(rs, 2 * nact, 1) for _ in range(nact)]
    desired = np.stack([rs.randint(0, nrow, nact), rs.randint(0, ncol, nact)], -1)
    pa = [K.nets.pack_padded(w, 2 * NA) for w in actors] + [K.nets.pack(rand_net(rs, 2 * NA, 5)) for _ in range(NA - nact)]
    pc = [K.nets.pack_padded(w, 2 * NA) for w in critics] + [K.nets.pack(rand_net(rs, 2 * NA, 1)) for _ in range(NA - nact)]
    des = np.zeros((NA, 2), np.int32)
    des[:nact] = desired
    dev = to_dev(K, np.stack(pa), np.stack(pc), des)
    draws = R.rollout_draws(seed, env_offset=env_off, n_envs=N, episode_offset=ep_off, n_episodes=N_EP, max_ep_len=LEN,
                            n_slots=NA, n_active=nact, nrow=nrow, ncol=ncol)
    return dict(actors=actors, critics=critics, desired=desired, dev=dev, draws=draws, scaling=nrow * ncol > 1)


def launch(K, case, st, injected):
    """One rcmarl_rollout into NaN-prefilled buffers with rows before time_begin and after the block."""
    NA, nact, nrow, ncol, N, env_off, ep_off, tb, mu, seed = case
    T = tb + N_EP * LEN + 2
    sa, ns, r = (torch.full((T * N, f * NA), NAN, device=K.dev) for f in (3, 2, 1))
    est, ret = (torch.full((N_EP, N, NA), NAN, device=K.dev) for _ in range(2))
    kw = {}
    if injected:
        dinit, dU = to_dev(K, *st["draws"])
        kw = dict(init_state=dinit, uniforms=dU)
    K.ops.rollout(*st["dev"], sa, ns, r, tb, est, ret, n_envs=N, n_agents=NA, n_episodes=N_EP, max_ep_len=LEN, nrow=nrow,
                  ncol=ncol, gamma=0.9, mu=mu, seed=seed, env_offset=env_off, episode_offset=ep_off, n_active=nact,
                  scaling=st["scaling"], **kw)
    torch.cuda.synchronize()
    return dict(sa=sa, ns=ns, r=r, est=est, ret=ret)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_philox_launch_equals_injected_restated_draws(K, case):
    """(a) Philox mode == injected mode fed rollout_draws(...), bit for bit in sa, ns, r, est, ret; the rows outside
    [time_begin, time_begin + n_ep * L) stay NaN and every row inside is written."""
    tb, N = case[7], case[4]
    st = setup_case(K, case)
    got, want = launch(K, case, st, injected=False), launch(K, case, st, injected=True)
    for name in got:
        assert torch.equal(got[name].view(torch.int32), want[name].view(torch.int32)), name
    for name in ("sa", "ns", "r"):
        x = got[name]
        assert torch.isnan(x[:tb * N]).all() and torch.isnan(x[(tb + N_EP * LEN) * N:]).all(), name
        assert not torch.isnan(x[tb * N:(tb + N_EP * LEN) * N]).any(), name
    for name in ("est", "ret"):
        assert not torch.isnan(got[name]).any()


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_philox_launch_matches_oracle(K, case):
    """(b) the Philox-mode launch against O.rollout_block in fp64 on the restated draws: rows exact outside ties,
    est / ret at the forward tolerances, the absent agent slots exact zeros."""
    NA, nact, nrow, ncol, N, env_off, ep_off, tb, mu, seed = case
    st = setup_case(K, case)
    got = launch(K, case, st, injected=False)
    agents = [O.RPBCACOracleAgent(st["actors"][i], st["critics"][i], rand_net(np.random.RandomState(i), 3 * nact, 1),
                                  0.002, 0.01, 0.9, dtype=f64) for i in range(nact)]
    want, est, ret = R.oracle_rollout(agents, st["desired"], nrow, ncol, st["draws"], 0.9, mu, st["scaling"])
    ok = R.check_rows(rows_of(got["sa"], got["ns"], got["r"], NA, nact, tb, tb + N_EP * LEN, N), want, N_EP, LEN, N)
    block = slice(tb * N, (tb + N_EP * LEN) * N)
    for name in ("sa", "ns", "r"):
        x = got[name][block].view(N_EP * LEN * N, NA, -1)[:, nact:]
        assert torch.equal(x, torch.zeros_like(x)), name
    for name in ("est", "ret"):
        x = got[name][..., nact:]
        assert torch.equal(x, torch.zeros_like(x)), name
    close(got["est"][..., :nact].cpu().numpy(), est, rtol=1e-5, atol=3e-6)       # est does not depend on actions
    close(got["ret"][..., :nact].cpu().numpy()[ok], ret[ok], rtol=1e-5, atol=1e-5)


# --------------------------------------------------------------------------------------------------- (c) bench block
def test_bench_first_block_matches_oracle(K):
    """(c) The first block bench.py rolls out: the C2 team (pretrained weights), 4096 environments, 50 episodes x 20
    steps, seed 1234, episode 0.  Rows against the fp64 oracle on the restated draws, and the per-episode means the
    Trainer returns (rcmarl_episode_means) against the fp64 means."""
    from rcmarl.trainer import Trainer
    w, desired, labels = pretrained()
    N, n_ep, L_ = 4096, 50, 20
    tr = Trainer(labels=labels, in_nodes=T16.IN5, weights=w, desired=desired, nrow=5, ncol=5, H=1, n_envs=N, gamma=0.9,
                 fast_lr=0.01, slow_lr=0.002, max_ep_len=L_, n_ep_fixed=n_ep, n_epochs=10, buffer_size=2000, seed=1234)
    est_m, ret_m = tr.rollout_block()
    agents = [O.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, 0.9, dtype=f64) for i in range(5)]
    draws = R.rollout_draws(1234, env_offset=0, n_envs=N, episode_offset=0, n_episodes=n_ep, max_ep_len=L_, n_slots=5,
                            n_active=5, nrow=5, ncol=5)
    want, est, ret = R.oracle_rollout(agents, desired, 5, 5, draws, 0.9)
    ok = R.check_rows(R.trainer_rows(tr, 0, n_ep * L_), want, n_ep, L_, N)
    close(est_m, est.mean(1), rtol=1e-5, atol=3e-6)
    full = ok.all(1)                                                      # episodes without a tie in any environment
    assert full.mean() > 0.5, full.mean()
    close(ret_m[full], ret[full].mean(1), rtol=1e-5, atol=1e-5)


# --------------------------------------------------------------------------------------------------- (d) training loop
LOOP = dict(gamma=0.9, max_ep_len=5, n_ep_fixed=4, n_epochs=2, buffer_size=30, slow_lr=0.002)   # buffer: 1.5 blocks
LOOP_SEED = 11          # the fp32 oracle stays within 1 % of the whole-round tolerance on every team below


@pytest.mark.parametrize("name,N", [("c2", 1), ("c2", 64), ("greedy_faulty", 16), ("M16", 8), ("team3_4x6", 16)])
def test_default_training_loop_matches_oracle(K, name, N):
    """(d) Three rollout blocks + update rounds of a Trainer with no injected draws, rows or shuffles, buffer_size =
    1.5 blocks (Phase IV trims from round 2 on), teacher-forced per round: before each block the oracle agents are
    loaded from the Trainer; the block's rows and logged means must be the oracle's rollout on the draws restated with
    episode_offset = episodes done and env_offset = rank x N; O.update_round on the Trainer's buffer with the
    Trainer's own shuffles (default_perm_source) must give its weights and losses; the kept buffer must be the newest
    buffer_size time rows."""
    from rcmarl.trainer import Trainer
    team = T16.loop_team(name)
    n = len(team["labels"])
    tr = Trainer(**team, n_envs=N, seed=LOOP_SEED, **LOOP)
    L_, ne, block = LOOP["max_ep_len"], LOOP["n_ep_fixed"], LOOP["max_ep_len"] * LOOP["n_ep_fixed"]
    perms = R.default_perm_source(LOOP_SEED)
    for k in range(3):
        assert tr.episodes_done == k * ne
        agents = R.oracle_agents_from_trainer(tr)
        draws = R.rollout_draws(LOOP_SEED, env_offset=tr.rank * N, n_envs=N, episode_offset=k * ne, n_episodes=ne,
                                max_ep_len=L_, n_slots=tr.NA, n_active=n, nrow=team["nrow"], ncol=team["ncol"])
        t0 = tr.t_filled
        est_m, ret_m = tr.rollout_block()
        want, est, ret = R.oracle_rollout(agents, team["desired"], team["nrow"], team["ncol"], draws, LOOP["gamma"])
        ok = R.check_rows(R.trainer_rows(tr, t0, t0 + block), want, ne, L_, N)
        close(est_m, est.mean(1), rtol=1e-5, atol=3e-6, err_msg=f"round {k} est")
        full = ok.all(1)
        close(ret_m[full], ret[full].mean(1), rtol=1e-5, atol=1e-5, err_msg=f"round {k} ret")

        buf = R.trainer_rows(tr, 0, tr.t_filled)
        got_loss = tr.update_round()
        want_loss = O.update_round(agents, team["labels"], team["in_nodes"], *buf, n_envs=N, n_epochs=LOOP["n_epochs"],
                                   n_actor_steps=block, common_reward=team.get("common_reward", False), perm_source=perms)
        for i in range(n):
            T16.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"round {k} agent {i}")
        for key in ("critic_loss", "TR_loss", "actor_loss"):
            np.testing.assert_allclose(got_loss[key], want_loss[key], rtol=2e-3, atol=2e-5, err_msg=f"round {k} {key}")
        keep = min(t0 + block, LOOP["buffer_size"])
        assert tr.t_filled == keep
        for g, x in zip(R.trainer_rows(tr, 0, keep), buf):
            assert np.array_equal(g, x[-keep * N:]), f"round {k}: kept buffer"


# --------------------------------------------------------------------------------------------------- (e) drop-in path
@pytest.mark.parametrize("n_envs", [1, 16])
def test_train_rpbcac_sim_data_matches_oracle(K, n_envs):
    """(e) training.train_RPBCAC as main.py calls it, n_episodes = n_ep_fixed + 3: the first block's sim_data rows are
    the reference's formulas (train_agents.py:168-180: team return = mean over the cooperative agents, adversary
    return = mean over the others, estimated return = mean of the cooperative agents' est) applied to the oracle's
    rollout at the initial weights; the 3 trailing episodes are the oracle's rollout at the returned weights with
    episode_offset = n_ep_fixed."""
    from rcmarl import api
    import training.train_agents as training
    w, desired, labels = pretrained()
    cfg = dict(labels=labels, in_nodes=T16.IN5, weights=w, desired=desired, nrow=5, ncol=5, H=1, n_envs=n_envs, gamma=0.9,
               fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=8, n_epochs=2, buffer_size=96)
    env, agents, args = api.build_reference_objects(cfg)
    ne, L_ = cfg["n_ep_fixed"], cfg["max_ep_len"]
    args["n_episodes"] = ne + 3
    weights, sim = training.train_RPBCAC(env, agents, args, verbose=False)
    tr = training.train_RPBCAC.last_trainer
    assert tr.episodes_done == ne + 3 and tr.t_filled == (ne + 3) * L_
    coop, adv = [i for i in range(5) if labels[i] == C], [i for i in range(5) if labels[i] != C]

    def block(ws, ep0, n_ep):
        ags = [O.RPBCACOracleAgent(ws[i][0], ws[i][1], ws[i][2], 0.002, 0.01, 0.9, dtype=f64) for i in range(5)]
        draws = R.rollout_draws(tr.seed, env_offset=0, n_envs=n_envs, episode_offset=ep0, n_episodes=n_ep, max_ep_len=L_,
                                n_slots=5, n_active=5, nrow=5, ncol=5)
        want, est, ret = R.oracle_rollout(ags, desired, 5, 5, draws, 0.9)
        ok = R.check_rows(R.trainer_rows(tr, ep0 * L_, (ep0 + n_ep) * L_), want, n_ep, L_, n_envs)
        assert ok.all()
        est, ret = est.mean(1), ret.mean(1)
        return np.stack([ret[:, coop].sum(1) / len(coop), ret[:, adv].sum(1) / len(adv), est[:, coop].mean(1)], 1)

    cols = ["True_team_returns", "True_adv_returns", "Estimated_team_returns"]
    got = sim[cols].to_numpy()
    close(got[:ne], block(w, 0, ne), rtol=1e-5, atol=1e-5)
    close(got[ne:], block(list(weights), ne, 3), rtol=1e-5, atol=1e-5)
