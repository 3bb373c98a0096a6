"""Teams shared by the trainer parity tests (test_trainer_gpu.py, test_dp_single_gpu.py, test_rollout_philox_gpu.py,
test_reference_scale_gpu.py): 16-agent teams with several adversaries on the 10x10 grid with circulant
in-neighbourhoods of 6, their fp64 oracle agents, seeded buffer rows, the oracle side of update rounds whose shuffles
the Trainer replays, and the Trainer configurations of the default-loop tests (loop_team)."""
import numpy as np

from golden_util import pretrained
from oracle import rpbcac_oracle as O

C, M, G, F = 'Cooperative', 'Malicious', 'Greedy', 'Faulty'
IN5 = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
TEAMS16 = {
    # 9 cooperative, 4 malicious, 2 greedy, 1 faulty agents: 4 x 3 + 2 x 2 = 16 mini-batch chains
    "M16": [C, M, C, G, C, M, C, F, C, M, C, G, C, M, C, C],
    # 5 cooperative + 11 malicious agents: 33 chains, one more than a kernel launch takes (RCMARL_MAX_JOBS)
    "X33": [C, M, M, C, M, M, C, M, M, C, M, M, C, M, M, M],
    # 16 malicious agents: 48 chains and no cooperative agent (no consensus, no projection, r_coop = 0)
    "A48": [M] * 16,
}


def team16(name, rs):
    """(labels, in_nodes, weights, desired, H, fast_lr) of TEAMS16[name]; weights and desired are drawn from rs.  Every
    agent has an H in {0, 1, 2} and a fast learning rate of its own, and every malicious agent its own critic_local net."""
    NA = 16
    labels = list(TEAMS16[name])
    in_nodes = [[(i + k) % NA for k in range(6)] for i in range(NA)]
    from rcmarl import nets
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    desired = rs.randint(0, 10, size=(NA, 2))
    local = np.random.RandomState(len(name) + sum(map(ord, name)))
    for i in range(NA):
        if labels[i] == M:
            w[i].append(nets.glorot_uniform(32, 1, local))
    return labels, in_nodes, w, desired, [i % 3 for i in range(NA)], [0.01 + 0.001 * (i % 4) for i in range(NA)]


def loop_team(name):
    """Trainer keywords (team, grid, H, fast_lr) of the default-loop tests: "c2" (the pretrained C2 team),
    "greedy_faulty" (its weights with agents 3, 4 Greedy and Faulty, common_reward), "M16" (team16) and any other name a
    padded 3-agent team on the 5-agent instantiation, 4 x 6 grid."""
    w, desired, labels = pretrained()
    if name == "c2":
        return dict(labels=labels, in_nodes=IN5, weights=w, desired=desired, nrow=5, ncol=5, H=1, fast_lr=0.01)
    if name == "greedy_faulty":
        return dict(labels=[C, C, C, G, F], in_nodes=IN5, weights=[x[:3] for x in w], desired=desired, nrow=5, ncol=5,
                    H=1, fast_lr=0.01, common_reward=True)
    if name == "M16":
        labels, in_nodes, w16, des, H, fast = team16("M16", np.random.RandomState(31))
        return dict(labels=labels, in_nodes=in_nodes, weights=w16, desired=des, nrow=10, ncol=10, H=H, fast_lr=fast)
    rs = np.random.RandomState(7)                                         # 3 agents on the 5-agent instantiation
    from rcmarl import nets
    w3 = [[nets.glorot_uniform(6, 5, rs), nets.glorot_uniform(6, 1, rs), nets.glorot_uniform(9, 1, rs)] for _ in range(3)]
    return dict(labels=[C, C, M], in_nodes=[[0, 1, 2], [1, 2, 0], [2, 0, 1]], weights=w3,
                desired=np.array([[1, 2], [3, 5], [0, 0]]), nrow=4, ncol=6, H=1, fast_lr=0.01)


def oracle_agents(labels, w, H, fast, gamma, slow_lr=0.002, dtype=np.float64):
    """Oracle agents (fp64 by default); a malicious agent without a critic_local net starts it from its critic (as
    Trainer does)."""
    ags = []
    for i, lab in enumerate(labels):
        a, c, t = w[i][0], w[i][1], w[i][2]
        if lab == C:
            ags.append(O.RPBCACOracleAgent(a, c, t, slow_lr, fast[i], gamma, H=H[i], dtype=dtype))
        elif lab == M:
            ags.append(O.MaliciousOracleAgent(a, c, t, slow_lr, fast[i], gamma,
                                              critic_local_w=w[i][3] if len(w[i]) > 3 else None, dtype=dtype))
        elif lab == G:
            ags.append(O.GreedyOracleAgent(a, c, t, slow_lr, fast[i], gamma, dtype=dtype))
        else:
            ags.append(O.FaultyOracleAgent(a, c, t, slow_lr, gamma, dtype=dtype))
    return ags


def grid_rows(rs, B, NA, nrow):
    """B transitions of NA agents on an nrow x nrow grid: scaled s / ns (one step apart), actions, rewards in [-(2 nrow
    - 2) / 5, 0]; s, ns: (B, NA, 2), a, r: (B, NA, 1) float32."""
    pos = rs.randint(0, nrow, size=(B, NA, 2))
    npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape), 0, nrow - 1)
    mean, std = (nrow - 1) / 2.0, np.std(np.arange(nrow))
    s = ((pos - mean) / std).astype(np.float32)
    ns = ((npos - mean) / std).astype(np.float32)
    a = rs.randint(0, 5, size=(B, NA, 1)).astype(np.float32)
    r = (-rs.randint(0, 2 * nrow - 1, size=(B, NA, 1)) / 5.0).astype(np.float32)
    return s, ns, a, r


class OracleRounds:
    """The oracle side of consecutive update rounds on a growing buffer (trimmed to its newest buffer_size time rows
    after each round, train_agents.py:158-163).  round() returns the oracle's losses and the time-row permutations it
    drew, in draw order, for the Trainer to replay."""

    def __init__(self, agents, labels, in_nodes, *, n_envs, n_epochs, n_actor_steps, buffer_size, perm_seed=4,
                 common_reward=False):
        self.agents, self.labels, self.in_nodes = agents, labels, in_nodes
        self.kw = dict(n_envs=n_envs, n_epochs=n_epochs, n_actor_steps=n_actor_steps, common_reward=common_reward)
        self.keep = buffer_size * n_envs
        self.rs = np.random.RandomState(perm_seed)
        self.buf = None

    def round(self, s, ns, a, r):
        new = (s, ns, a, r)
        self.buf = new if self.buf is None else tuple(np.concatenate([x, y]) for x, y in zip(self.buf, new))
        used = []

        def rec(T):
            p = self.rs.permutation(T)
            used.append(p)
            return p
        loss = O.update_round(self.agents, self.labels, self.in_nodes, *self.buf, perm_source=rec, **self.kw)
        self.buf = tuple(x[-self.keep:] for x in self.buf)
        return loss, used


class Replay:
    """perm_source for Trainer: hands out the oracle's permutations in order (load() appends a round's)."""

    def __init__(self):
        self.perms = []

    def load(self, perms):
        self.perms.extend(perms)

    def __call__(self, T):
        p = self.perms.pop(0)
        assert len(p) == T
        return p

    def done(self):
        return not self.perms


def close_w(got, want, rtol=1e-3, atol=5e-5, msg=""):
    for n in range(len(want)):
        for k in range(6):
            np.testing.assert_allclose(np.asarray(got[n][k], np.float64), np.asarray(want[n][k], np.float64),
                                       rtol=rtol, atol=atol, err_msg=f"{msg} net {n} array {k}")
