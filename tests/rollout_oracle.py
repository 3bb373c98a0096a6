"""The random streams of rcmarl_rollout's Philox branch, restated from include/rcmarl.h (not from the kernel), and the
pieces that let the fp64 oracle (oracle/rpbcac_oracle.py) follow the Trainer's default training loop round by round:

  rollout_draws          the reset positions and action uniforms a Philox-mode launch draws, in the layout of the
                         injected branch and of O.rollout_block;
  reset_counters / action_counters
                         their Philox counters (also used to check that the streams never share a counter);
  default_perm_source    the Trainer's own mini-batch shuffles (perm_source=None);
  oracle_agents_from_trainer / trainer_rows
                         oracle agents and buffer rows read back from a Trainer.

Philox4x32-10 itself is attack_oracle.philox4x32_10 (integer-exact, checked against the Random123 known answers)."""
import numpy as np

from attack_oracle import philox4x32_10
from oracle import rpbcac_oracle as O

M32 = 0xFFFFFFFF
RESET_BIT = 0x80000000                     # word 1 of every reset counter
ATTACK_BIT = 0x40000000                    # word 1 of every rcmarl_attack counter (bit 31 clear)
U01 = np.float32(2.0 ** -24)


def _key(seed):
    seed = int(seed)
    return seed & M32, (seed >> 32) & M32


def _env_words(env_offset, n_envs):
    g = int(env_offset) + np.arange(n_envs, dtype=np.uint64)
    return g & np.uint64(M32), g >> np.uint64(32)


def _episode_words(episode_offset, n_episodes):
    return (int(episode_offset) + np.arange(n_episodes, dtype=np.uint64)) & np.uint64(M32)


def reset_counters(*, env_offset, n_envs, episode_offset, n_episodes, n_active):
    """Counter words of the reset draws, each [n_episodes][n_envs][n_active]:
    (g low, g high ^ 0x80000000, episode word, agent) with g = env_offset + env."""
    lo, hi = _env_words(env_offset, n_envs)
    ep = _episode_words(episode_offset, n_episodes)
    shape = (n_episodes, n_envs, n_active)
    return [np.broadcast_to(lo[None, :, None], shape), np.broadcast_to((hi ^ np.uint64(RESET_BIT))[None, :, None], shape),
            np.broadcast_to(ep[:, None, None], shape), np.broadcast_to(np.arange(n_active, dtype=np.uint64), shape)]


def action_counters(*, env_offset, n_envs, episode_offset, n_episodes, max_ep_len, n_slots, n_active):
    """Counter words of the action draws, each [n_episodes][max_ep_len][n_envs][n_active]:
    (g low, g high, episode word, step * n_slots + agent); n_slots is the kernel instantiation (5 or 16)."""
    lo, hi = _env_words(env_offset, n_envs)
    ep = _episode_words(episode_offset, n_episodes)
    shape = (n_episodes, max_ep_len, n_envs, n_active)
    w3 = np.arange(max_ep_len, dtype=np.uint64)[:, None] * np.uint64(n_slots) + np.arange(n_active, dtype=np.uint64)
    return [np.broadcast_to(lo[None, None, :, None], shape), np.broadcast_to(hi[None, None, :, None], shape),
            np.broadcast_to(ep[:, None, None, None], shape), np.broadcast_to(w3[None, :, None, :], shape)]


def u01(w):
    """(w >> 8) * 2^-24: 24 random bits, exact in fp32, in [0, 1)."""
    return (np.asarray(w, np.uint32) >> np.uint32(8)).astype(np.float32) * U01


def rollout_draws(seed, *, env_offset, n_envs, episode_offset, n_episodes, max_ep_len, n_slots, n_active, nrow, ncol):
    """What a Philox-mode rcmarl_rollout draws: (init_states int32 [n_ep][N][n_active][2],
    uniforms float32 [n_ep][L][N][n_active][3]), exactly the arrays its injected branch and O.rollout_block take.
    Resets: px = umulhi(x, nrow), py = umulhi(y, ncol); actions: u0, u1, u2 = u01(x), u01(y), u01(z)."""
    key = _key(seed)
    init = np.empty((n_episodes, n_envs, n_active, 2), np.int32)
    uni = np.empty((n_episodes, max_ep_len, n_envs, n_active, 3), np.float32)
    for e in range(n_episodes):                         # one episode at a time bounds the uint64 temporaries
        kw = dict(env_offset=env_offset, n_envs=n_envs, episode_offset=int(episode_offset) + e, n_episodes=1)
        x, y, _, _ = philox4x32_10(reset_counters(n_active=n_active, **kw), key)
        init[e, ..., 0] = (x[0].astype(np.uint64) * np.uint64(nrow)) >> np.uint64(32)
        init[e, ..., 1] = (y[0].astype(np.uint64) * np.uint64(ncol)) >> np.uint64(32)
        x, y, z, _ = philox4x32_10(action_counters(max_ep_len=max_ep_len, n_slots=n_slots, n_active=n_active, **kw), key)
        uni[e, ..., 0], uni[e, ..., 1], uni[e, ..., 2] = u01(x[0]), u01(y[0]), u01(z[0])
    return init, uni


def default_perm_source(seed):
    """The Trainer's shuffles with perm_source=None: torch.randperm(T, int32) from a CPU generator seeded
    seed * 7919 + 17, called in the Trainer's draw order (which is the oracle's)."""
    import torch
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed) * 7919 + 17)
    return lambda T: torch.randperm(T, generator=g, dtype=torch.int32).numpy()


def oracle_agents_from_trainer(tr, dtype=np.float64):
    """Oracle agents holding the Trainer's current state (tr.state_dict()): actor / critic / TR weights, the Malicious
    agents' critic_local, and the Keras-Adam m, v, t of every actor, with the Trainer's per-agent H, fast_lr, slow_lr."""
    from rcmarl import nets
    sd = tr.state_dict(include_buffer=False)
    n, NA = tr.n_real, tr.NA

    def net(name, i, f, n_out):
        return nets.unpack_padded(sd[name][i].numpy(), f * n, f * NA, n_out)
    agents = []
    for i in range(n):
        lab = tr.labels[i]
        a, c, t = net("actor", i, 2, 5), net("critic", i, 2, 1), net("tr", i, 3, 1)
        if lab == "Cooperative":
            ag = O.RPBCACOracleAgent(a, c, t, tr.slow_lr[i], tr.fast_lr[i], tr.gamma, H=tr.H[i], dtype=dtype)
        elif lab == "Malicious":
            ag = O.MaliciousOracleAgent(a, c, t, tr.slow_lr[i], tr.fast_lr[i], tr.gamma,
                                        critic_local_w=net("critic_local", i, 2, 1), dtype=dtype)
        elif lab == "Greedy":
            ag = O.GreedyOracleAgent(a, c, t, tr.slow_lr[i], tr.fast_lr[i], tr.gamma, dtype=dtype)
        elif lab == "Faulty":
            ag = O.FaultyOracleAgent(a, c, t, tr.slow_lr[i], tr.gamma, dtype=dtype)
        else:
            raise ValueError(f"no oracle agent for label {lab!r}")
        steps = int(sd["adam_t"][i])
        if steps:
            ag.adam.m = [x.astype(dtype) for x in net("adam_m", i, 2, 5)]
            ag.adam.v = [x.astype(dtype) for x in net("adam_v", i, 2, 5)]
            ag.adam.t = steps
        agents.append(ag)
    return agents


def trainer_rows(tr, t0, t1):
    """Time rows [t0, t1) of the Trainer's buffer for its real agents as float32 arrays in the oracle's layout:
    s, ns (B, n, 2) and a, r (B, n, 1), B = (t1 - t0) * n_envs."""
    n, NA, N = tr.n_real, tr.NA, tr.N
    lo, hi = t0 * N, t1 * N
    sa = tr.sa[lo:hi].view(-1, NA, 3)[:, :n].cpu().numpy()
    ns = tr.ns[lo:hi].view(-1, NA, 2)[:, :n].cpu().numpy()
    r = tr.r[lo:hi].view(-1, NA, 1)[:, :n].cpu().numpy()
    return sa[:, :, :2].copy(), ns, sa[:, :, 2:].copy(), r
