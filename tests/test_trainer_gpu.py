"""GPU parity of the batched training engine (rcmarl.trainer.Trainer) against
 (a) the golden run of the reference's own train_RPBCAC executed verbatim on the facade
     (tests/golden/ref_train_run.npz: 2 update rounds, 4 cooperative + 1 malicious, H=1), and
 (b) the CPU oracle on a batched (n_envs > 1) configuration incl. Greedy / Faulty agents.
Tolerance: weights after full update rounds rtol 1e-3 / atol 5e-5 (hundreds of chained fp32 SGD steps;
single steps are held to 1e-4 in test_kernels_gpu.py)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from golden_util import load, agent_weights, pretrained    # noqa: E402
import team_util as T16                                      # noqa: E402
from oracle import rpbcac_oracle as O                        # noqa: E402

IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def close_w(got, want, rtol=1e-3, atol=5e-5):
    for n in range(len(want)):
        for k in range(6):
            np.testing.assert_allclose(np.asarray(got[n][k], np.float64), np.asarray(want[n][k], np.float64),
                                       rtol=rtol, atol=atol, err_msg=f"net {n} array {k}")


def test_two_update_rounds_match_reference_train_run():
    need_gpu()
    from rcmarl.trainer import Trainer
    z = load("ref_train_run.npz")
    w, desired, labels = pretrained()
    perms = [z[f"perm{j}"] for j in range(int(z["n_perms"]))]
    it = iter(perms)

    def perm_source(T):
        p = next(it)
        assert len(p) == T
        return p
    tr = Trainer(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=1, gamma=0.9, H=1, fast_lr=0.01,
                 slow_lr=0.002, max_ep_len=10, n_ep_fixed=25, n_epochs=2, buffer_size=100000, capacity_times=600,
                 perm_source=perm_source)
    for rnd in (0, 1):
        sl = slice(250 * rnd, 250 * (rnd + 1))
        tr.load_rows(z["s"][sl], z["ns"][sl], z["a"][sl], z["r"][sl])
        tr.update_round()
    assert next(it, None) is None
    final = agent_weights(z, "final")
    for i in range(5):
        close_w(tr.get_weights(i), final[i])


@pytest.mark.parametrize("labels,common,H", [
    (['Cooperative'] * 5, False, 0),
    (['Cooperative', 'Cooperative', 'Cooperative', 'Greedy', 'Faulty'], True, 1),
    (['Cooperative', 'Cooperative', 'Cooperative', 'Cooperative', 'Malicious'], False, 1),
    (['Cooperative', 'Cooperative', 'Cooperative', 'Malicious', 'Malicious'], False, 1)])
def test_batched_update_round_matches_oracle(labels, common, H):
    need_gpu()
    from rcmarl.trainer import Trainer
    rs = np.random.RandomState(3)
    N, T1, gamma = 6, 48, 0.9
    w, desired, _ = pretrained()

    def make_oracle():
        ags = []
        for i, l in enumerate(labels):
            a, c, t = w[i][0], w[i][1], w[i][2]
            if l == 'Cooperative':
                ags.append(O.RPBCACOracleAgent(a, c, t, 0.002, 0.01, gamma, H=H, dtype=np.float64))
            elif l == 'Malicious':
                ags.append(O.MaliciousOracleAgent(a, c, t, 0.002, 0.01, gamma, critic_local_w=w[i][3] if len(w[i]) > 3 else None,
                                                   dtype=np.float64))
            elif l == 'Greedy':
                ags.append(O.GreedyOracleAgent(a, c, t, 0.002, 0.01, gamma, dtype=np.float64))
            else:
                ags.append(O.FaultyOracleAgent(a, c, t, 0.002, gamma, dtype=np.float64))
        return ags
    agents = make_oracle()
    rs_perm = np.random.RandomState(4)
    used = []

    def perm_rec(T):
        p = rs_perm.permutation(T)
        used.append(p)
        return p
    it = None

    def perm_replay(T):
        p = next(it)
        assert len(p) == T
        return p
    tr = Trainer(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=H, fast_lr=0.01,
                 slow_lr=0.002, max_ep_len=8, n_ep_fixed=6, n_epochs=2, buffer_size=64, common_reward=common,
                 perm_source=perm_replay)
    S = NS = A = R = None
    for rnd in range(2):
        B = T1 * N
        pos = rs.randint(0, 5, size=(B, 5, 2))
        npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape), 0, 4)
        s = ((pos - 2.0) / np.std(np.arange(5))).astype(np.float32)
        ns = ((npos - 2.0) / np.std(np.arange(5))).astype(np.float32)
        a = rs.randint(0, 5, size=(B, 5, 1)).astype(np.float32)
        r = (-rs.randint(0, 9, size=(B, 5, 1)) / 5.0).astype(np.float32)
        S, NS, A, R = (s, ns, a, r) if S is None else tuple(np.concatenate([x, y]) for x, y in ((S, s), (NS, ns), (A, a), (R, r)))
        used.clear()
        want_loss = O.update_round(agents, labels, IN_NODES, S, NS, A, R, n_envs=N, n_epochs=2, n_actor_steps=48,
                                   common_reward=common, perm_source=perm_rec)
        it = iter(list(used))
        tr.load_rows(s, ns, a, r)
        got_loss = tr.update_round()
        assert next(it, None) is None
        for k in ("critic_loss", "TR_loss", "actor_loss"):
            np.testing.assert_allclose(got_loss[k], want_loss[k], rtol=2e-3, atol=2e-5, err_msg=k)
        # oracle-side trim (train_agents.py:158-163): newest 64 time rows
        keep = 64 * N
        S, NS, A, R = S[-keep:], NS[-keep:], A[-keep:], R[-keep:]
        assert tr.t_filled == min(64, T1 * (rnd + 1))
        np.testing.assert_array_equal(tr.ns[:tr.t_filled * N].cpu().numpy().reshape(-1, 5, 2), NS)
    for i in range(5):
        close_w(tr.get_weights(i), agents[i].get_parameters())


def test_checkpoint_resume_is_bitwise(tmp_path):
    """state_dict / load_state_dict: weights, Adam slots, buffer, Philox episode counter and shuffle stream -- a resumed
    run continues exactly like the uninterrupted one (the reference cannot resume optimiser state or buffer)."""
    need_gpu()
    from rcmarl.trainer import Trainer
    w, desired, labels = pretrained()
    kw = dict(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=32, gamma=0.9, H=1, fast_lr=0.01,
              slow_lr=0.002, max_ep_len=6, n_ep_fixed=7, n_epochs=2, buffer_size=60, seed=9)
    a = Trainer(**kw)
    a.rollout_block(); a.update_round()
    a.save(tmp_path / "ckpt.pt")
    a.rollout_block(); a.update_round()
    b = Trainer(**kw)
    b.load(tmp_path / "ckpt.pt")
    assert b.t_filled == 42 and b.adam_t == [1] * 5
    b.rollout_block(); b.update_round()
    for name in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v", "sa", "ns", "r"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert a.adam_t == b.adam_t and a.episodes_done == b.episodes_done


def test_c3_shape_update_round_matches_oracle():
    """BASELINE config 3 shape at test size: 10x10 grid, 16 cooperative agents, H = 2, circulant in-neighbourhoods of 6
    (SURVEY 8d), batched environments -- the n_agents = 16 instantiation of every kernel through the trainer."""
    need_gpu()
    from rcmarl.trainer import Trainer
    from rcmarl import nets
    rs = np.random.RandomState(11)
    NA, N, T1, gamma, H = 16, 3, 40, 0.9, 2
    labels = ['Cooperative'] * NA
    in_nodes = [[(i + k) % NA for k in range(6)] for i in range(NA)]
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    desired = rs.randint(0, 10, size=(NA, 2))
    agents = [O.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, H=H, dtype=np.float64) for i in range(NA)]
    tr = Trainer(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma, H=H,
                 fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100)
    B = T1 * N
    pos = rs.randint(0, 10, size=(B, NA, 2))
    npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape), 0, 9)
    mean, std = 4.5, np.std(np.arange(10))
    s = ((pos - mean) / std).astype(np.float32)
    ns = ((npos - mean) / std).astype(np.float32)
    a = rs.randint(0, 5, size=(B, NA, 1)).astype(np.float32)
    r = (-rs.randint(0, 19, size=(B, NA, 1)) / 5.0).astype(np.float32)
    want = O.update_round(agents, labels, in_nodes, s, ns, a, r, n_envs=N, n_epochs=2, n_actor_steps=40,
                          common_reward=False, perm_source=lambda T: np.arange(T))
    tr.load_rows(s, ns, a, r)
    got = tr.update_round()
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(NA):
        close_w(tr.get_weights(i), agents[i].get_parameters())


# The seeds give data on which the fp32 oracle itself stays within 1 % of the tolerance: with several adversaries among
# the neighbours, the clipped means make some data sets so ill-conditioned that fp32 arithmetic alone misses the fp64
# weights by more than the tolerance.
@pytest.mark.parametrize("team,seed", [("M16", 23), ("X33", 18), ("A48", 20)])
def test_c3_shape_adversarial_update_rounds_match_oracle(team, seed):
    """The C3 shape of test_c3_shape_update_round_matches_oracle (10x10 grid, 16 agents, circulant in-neighbourhoods of
    6) with several adversaries (tests/team_util.py), so tdt_local has several rows and one persistent launch runs several
    adversaries' chains: M16 mixes every agent kind at per-agent H and fast_lr (16 chains), X33 has 33 chains and A48 48
    chains without any cooperative agent -- more than one launch takes, so the trainer fits them in groups.  Two rounds
    at 4 environments: the second fits 80 time rows (a short third mini-batch)."""
    need_gpu()
    from rcmarl.trainer import Trainer
    rs = np.random.RandomState(seed)
    NA, N, T1, gamma = 16, 4, 40, 0.9
    labels, in_nodes, w, desired, H, fast = T16.team16(team, rs)
    agents = T16.oracle_agents(labels, w, H, fast, gamma)
    oracle = T16.OracleRounds(agents, labels, in_nodes, n_envs=N, n_epochs=2, n_actor_steps=40, buffer_size=100)
    replay = T16.Replay()
    tr = Trainer(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma, H=H,
                 fast_lr=fast, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, perm_source=replay)
    for _ in range(2):
        s, ns, a, r = T16.grid_rows(rs, T1 * N, NA, 10)
        want, perms = oracle.round(s, ns, a, r)
        replay.load(perms)
        tr.load_rows(s, ns, a, r)
        got = tr.update_round()
        assert replay.done()
        for k in ("critic_loss", "TR_loss", "actor_loss"):
            np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(NA):
        close_w(tr.get_weights(i), agents[i].get_parameters())


def test_env_options_scaling_off_and_fixed_initial_state():
    """Grid_World(scaling=False, randomize_state=False, initial_state=...) of the reference (grid_world.py:21-45): the
    rollout feeds raw integer positions and every episode starts from initial_state; nrow > ncol keeps both
    coordinates clipped with nrow - 1 (:55) and scaled with their own axis statistics."""
    need_gpu()
    from rcmarl.trainer import Trainer
    from rcmarl import ops
    w, desired, labels = pretrained()
    init = np.array([[0, 1], [4, 4], [2, 3], [1, 0], [3, 2]])
    tr = Trainer(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=16, gamma=0.9, H=1, max_ep_len=6,
                 n_ep_fixed=4, n_epochs=1, buffer_size=100, scaling=False, fixed_initial_state=init)
    tr.rollout_block()
    sa = tr.sa[:4 * 6 * 16].cpu().numpy().reshape(4, 6, 16, 5, 3)
    assert np.array_equal(sa[:, 0, :, :, :2], np.broadcast_to(init.astype(np.float32), (4, 16, 5, 2)))
    assert set(np.unique(sa[..., :2])) <= {0.0, 1.0, 2.0, 3.0, 4.0}
    tx, ty = ops.state_tables(7, 4)
    assert len(tx) == len(ty) == 7 and np.isclose(ty[6], (6 - 1.5) / np.std(np.arange(4)))
    tall = Trainer(labels=labels, in_nodes=IN_NODES, weights=w, desired=np.minimum(desired, 3), n_envs=64, nrow=7, ncol=4,
                   gamma=0.9, H=1, max_ep_len=20, n_ep_fixed=6, n_epochs=1, buffer_size=200, seed=3)
    tall.rollout_block()
    ns_y = tall.ns[:20 * 6 * 64].cpu().numpy().reshape(-1, 5, 2)[:, :, 1]
    assert set(np.unique(ns_y)) <= set(ty.tolist())          # no zero table entries: every reachable y is scaled
    assert ns_y.max() > ty[3] + 1e-6                          # ... and y does leave [0, ncol)


@pytest.mark.parametrize("NA,nrow,Hs", [(3, 3, [1, 1, 1]), (4, 5, [0, 1, 1, 0]), (7, 6, [2, 1, 2, 0, 1, 2, 1])])
def test_other_team_sizes_and_per_agent_H_match_oracle(NA, nrow, Hs):
    """main.py:26 takes any --n_agents (the reference's env_test.py uses 3 agents on a 3x3 grid) and the reference stores H
    and fast_lr per agent (agents/resilient_CAC_agents.py:28-36).  Teams of 3 / 4 / 7 agents run on the 5- / 16-agent kernel
    instantiations with zero agent slots; every agent has its own H and fast learning rate; one agent is greedy."""
    need_gpu()
    from rcmarl.trainer import Trainer
    from rcmarl import nets
    rs = np.random.RandomState(NA)
    N, T1, gamma = 6, 40, 0.9
    labels = ['Cooperative'] * NA
    labels[-1] = 'Greedy'
    n_in = min(NA, 4)
    in_nodes = [[(i + k) % NA for k in range(n_in)] for i in range(NA)]
    fast = [0.01 + 0.002 * i for i in range(NA)]
    w = [[nets.glorot_uniform(2 * NA, 5, rs), nets.glorot_uniform(2 * NA, 1, rs), nets.glorot_uniform(3 * NA, 1, rs)] for _ in range(NA)]
    desired = rs.randint(0, nrow, size=(NA, 2))
    agents = []
    for i in range(NA):
        if labels[i] == 'Greedy':
            agents.append(O.GreedyOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, fast[i], gamma, dtype=np.float64))
        else:
            agents.append(O.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, fast[i], gamma, H=Hs[i], dtype=np.float64))
    used = []
    prs = np.random.RandomState(5)

    def rec(T):
        p = prs.permutation(T)
        used.append(p)
        return p
    B = T1 * N
    pos = rs.randint(0, nrow, size=(B, NA, 2))
    npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape), 0, nrow - 1)
    mean, std = (nrow - 1) / 2.0, np.std(np.arange(nrow))
    s = ((pos - mean) / std).astype(np.float32)
    ns = ((npos - mean) / std).astype(np.float32)
    a = rs.randint(0, 5, size=(B, NA, 1)).astype(np.float32)
    r = (-rs.randint(0, 2 * nrow, size=(B, NA, 1)) / 5.0).astype(np.float32)
    want = O.update_round(agents, labels, in_nodes, s, ns, a, r, n_envs=N, n_epochs=2, n_actor_steps=T1,
                          common_reward=False, perm_source=rec)
    it = iter(list(used))
    tr = Trainer(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=nrow, ncol=nrow, gamma=gamma,
                 H=Hs, fast_lr=fast, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100,
                 perm_source=lambda T: next(it))
    tr.load_rows(s, ns, a, r)
    got = tr.update_round()
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k][:NA], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(NA):
        gw = tr.get_weights(i)
        assert gw[0][0].shape == (2 * NA, 20) and gw[2][0].shape == (3 * NA, 20)
        close_w(gw, agents[i].get_parameters())
    # the unused agent slots stayed exactly zero (inputs, W1 rows, Adam slots)
    NK = tr.NA
    assert float(tr.tr[:NA].view(NA, -1)[:, 3 * NA * 20:3 * NK * 20].abs().max()) == 0.0
    assert float(tr.actor[:NA].view(NA, -1)[:, 2 * NA * 20:2 * NK * 20].abs().max()) == 0.0
    # and a rollout block only moves the real agents
    e, rt = tr.rollout_block()
    assert e.shape == (5, NA) and rt.shape == (5, NA)
    rows = tr.sa[tr.t_filled * N - 8 * 5 * N:tr.t_filled * N].view(-1, NK, 3)
    assert float(rows[:, NA:].abs().max()) == 0.0 and float(rows[:, :NA, :2].abs().max()) > 0.0
