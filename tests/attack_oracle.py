"""Byzantine messages crafted per receiver (rcmarl_attack, include/rcmarl.h) on top of the NumPy oracle
(oracle/rpbcac_oracle.py), in the oracle's dtype (fp32 or fp64): the honest mean / population std and the three
attacks, the Philox4x32-10 counter layout and Box-Muller of the Gaussian attack (integer-exact), the hook that builds
each receiver's message list, and the oracle's update round with that hook.

update_round is O.update_round with one optional keyword, messages_hook, called after the Phase-I loop of every epoch;
it also treats a "Byzantine" agent as the oracle's Faulty one (both learn only their actor).  With messages_hook=None
and the reference's labels it computes what O.update_round computes (test_attacks_cpu.py checks that bit for bit), so
the oracle itself stays unchanged."""
import numpy as np

from oracle import rpbcac_oracle as O

ATTACKS = ("alie", "ipm", "gauss")
M32 = np.uint64(0xFFFFFFFF)


# ------------------------------------------------------------------------------------------------ Philox / Box-Muller
def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al. 2011), as csrc/common.cuh.  ctr: 4 uint32 words (scalars or arrays of one shape),
    key: 2 uint32 words -> 4 uint32 arrays.  Integer-exact: the products are formed in uint64."""
    c = [np.asarray(x, np.uint64) & M32 for x in ctr]
    k0, k1 = np.uint64(key[0]) & M32, np.uint64(key[1]) & M32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & M32, p1 & M32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & M32, p0 & M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return [x.astype(np.uint32) for x in c]


def counter(n, attacker, receiver, round_, epoch):
    """The counter words of coordinates 0..n-1: (p, attacker | receiver << 8 | 0x40000000, round, epoch)."""
    p = np.arange(n, dtype=np.uint64)
    w1 = (int(attacker) | int(receiver) << 8 | 0x40000000) & 0xFFFFFFFF
    return [p, np.full(n, w1, np.uint64), np.full(n, int(round_) & 0xFFFFFFFF, np.uint64),
            np.full(n, int(epoch) & 0xFFFFFFFF, np.uint64)]


def gauss_xi(n, seed, attacker, receiver, round_, epoch, dtype=np.float64):
    """xi_p ~ N(0, 1) for p < n: u1 = ((x >> 8) + 1) 2^-24, u2 = (y >> 8) 2^-24 (both exact in fp32),
    xi = sqrt(-2 ln u1) cos(2 pi u2) in `dtype`."""
    seed, dtype = int(seed), np.dtype(dtype).type
    x, y, _, _ = philox4x32_10(counter(n, attacker, receiver, round_, epoch), (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    u1 = ((x >> np.uint32(8)).astype(np.float64) + 1.0) * 2.0 ** -24
    u2 = (y >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    u1, u2 = u1.astype(dtype), u2.astype(dtype)
    return (np.sqrt(dtype(-2) * np.log(u1)) * np.cos(dtype(2 * np.pi) * u2)).astype(dtype)


# ------------------------------------------------------------------------------------------------ the attacks
def moments(values):
    """mu, sigma over axis 0 of values [n, P] in values' dtype: the mean summed in row order, the population std in
    two passes."""
    v = np.asarray(values)
    n = v.dtype.type(v.shape[0])
    s = np.zeros(v.shape[1:], v.dtype)
    for k in range(v.shape[0]):
        s = s + v[k]
    mu = s / n
    q = np.zeros(v.shape[1:], v.dtype)
    for k in range(v.shape[0]):
        q = q + (v[k] - mu) * (v[k] - mu)
    return mu, np.sqrt(q / n)


def craft(values, kind, param, xi=None):
    """The message of `kind` with parameter `param` against the honest messages values [n, P] (packed parameters);
    xi [P] is the Gaussian draw of "gauss"."""
    v = np.asarray(values)
    dt = v.dtype.type
    mu, sigma = moments(v)
    if kind == "alie":
        return mu - dt(param) * sigma
    if kind == "ipm":
        return -dt(param) * mu
    if kind == "gauss":
        if not param >= 0:
            raise ValueError("gauss needs s >= 0")
        return mu + dt(param) * np.asarray(xi, v.dtype)
    raise ValueError(f"unknown attack {kind!r}")


def pack(w, dtype):
    return np.concatenate([np.asarray(a, dtype).reshape(-1) for a in w])


def unpack(flat, like):
    out, o = [], 0
    for a in like:
        a = np.asarray(a)
        out.append(flat[o:o + a.size].reshape(a.shape))
        o += a.size
    return out


def byzantine_pairs(labels, in_nodes):
    """[(attacker b, cooperative receiver j, honest set S_j)] in the Trainer's order: b ascending, then j ascending."""
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    pairs = []
    for b, l in enumerate(labels):
        if l != "Byzantine":
            continue
        for j in coop:
            if b in in_nodes[j]:
                pairs.append((b, j, [k for k in in_nodes[j] if labels[k] == "Cooperative"]))
    return pairs


def make_hook(labels, in_nodes, attacks, seed=0, round_=0):
    """messages_hook of update_round: every cooperative receiver gets its own message list, in which each Byzantine
    neighbour's entry is crafted from the receiver's honest set in this epoch.  attacks[b] = (name, param)."""
    pairs = byzantine_pairs(labels, in_nodes)

    def hook(epoch, critic_msgs, TR_msgs):
        dt = critic_msgs[0][0].dtype
        per_c = {j: [critic_msgs[i] for i in in_nodes[j]] for j in range(len(labels))}
        per_t = {j: [TR_msgs[i] for i in in_nodes[j]] for j in range(len(labels))}
        for b, j, honest in pairs:
            kind, param = attacks[b]
            for msgs, per in ((critic_msgs, per_c), (TR_msgs, per_t)):
                vals = np.stack([pack(msgs[k], dt) for k in honest])
                xi = gauss_xi(vals.shape[1], seed, b, j, round_, epoch, dt) if kind == "gauss" else None
                m = unpack(craft(vals, kind, param, xi), msgs[b])
                per[j] = [m if i == b else x for i, x in zip(in_nodes[j], per[j])]
        return per_c, per_t
    return hook


# ------------------------------------------------------------------------------------------------ update round
def update_round(agents, labels, in_nodes, s, ns, a, r, *, n_envs, n_epochs, n_actor_steps,
                 common_reward, perm_source, messages_hook=None):
    """O.update_round (training/train_agents.py:86-163) with messages_hook(epoch, critic_msgs, TR_msgs) ->
    (critic lists, TR lists) per receiver, called after the Phase-I loop of every epoch; None: receiver j gets the
    messages of in_nodes[j]."""
    n_agents = len(agents)
    dt = agents[0].dtype
    s = np.asarray(s, dt)
    ns = np.asarray(ns, dt)
    a = np.asarray(a, dt)
    r = np.asarray(r, dt)
    B = s.shape[0]
    T = B // n_envs
    sa = np.concatenate([s, a], axis=-1)
    coop = [i for i in range(n_agents) if labels[i] == 'Cooperative']
    n_coop = len(coop)
    r_coop = np.zeros((B, 1), dt)
    for node in coop:
        r_coop = r_coop + r[:, node] / dt(n_coop)
    critic_loss = np.zeros(n_agents)
    TR_loss = np.zeros(n_agents)
    actor_loss = np.zeros(n_agents)

    def perms(n_ep):
        return [O.expand_time_perm(perm_source(T), n_envs) for _ in range(n_ep)]

    bs = 32 * n_envs
    for epoch in range(n_epochs):
        critic_msgs, TR_msgs = [], []
        for node in range(n_agents):
            r_applied = r_coop if common_reward else r[:, node]
            lab = labels[node]
            if lab == 'Cooperative':
                x, TR_loss[node] = agents[node].TR_update_local(sa, r_applied)
                y, critic_loss[node] = agents[node].critic_update_local(s, ns, r_applied)
            elif lab == 'Greedy':
                x, TR_loss[node] = agents[node].TR_update_local(sa, r[:, node], perms(10), bs)
                y, critic_loss[node] = agents[node].critic_update_local(s, ns, r[:, node], perms(10), bs)
            elif lab == 'Malicious':
                agents[node].critic_update_local(s, ns, r[:, node], perms(10), bs)
                x, TR_loss[node] = agents[node].TR_update_compromised(sa, -r_coop, perms(10), bs)
                y, critic_loss[node] = agents[node].critic_update_compromised(s, ns, -r_coop, perms(10), bs)
            elif lab in ('Faulty', 'Byzantine'):
                x = agents[node].get_TR_weights()
                y = agents[node].get_critic_weights()
            TR_msgs.append(x)
            critic_msgs.append(y)
        if messages_hook is None:
            per_c = {j: [critic_msgs[i] for i in in_nodes[j]] for j in coop}
            per_t = {j: [TR_msgs[i] for i in in_nodes[j]] for j in coop}
        else:
            per_c, per_t = messages_hook(epoch, critic_msgs, TR_msgs)
        for node in coop:
            cm, tm = per_c[node], per_t[node]
            agents[node].resilient_consensus_critic_hidden(cm)
            agents[node].resilient_consensus_TR_hidden(tm)
            critic_agg = agents[node].resilient_consensus_critic(s, cm)
            TR_agg = agents[node].resilient_consensus_TR(sa, tm)
            agents[node].critic_update_team(s, critic_agg)
            agents[node].TR_update_team(sa, TR_agg)
    na = n_actor_steps * n_envs
    Ta = n_actor_steps
    for node in range(n_agents):
        if labels[node] == 'Cooperative':
            actor_loss[node] = agents[node].actor_update(s[-na:], ns[-na:], sa[-na:], a[-na:, node])
        else:
            perm = O.expand_time_perm(perm_source(min(Ta, T)), n_envs)
            actor_loss[node] = agents[node].actor_update(s[-na:], ns[-na:], r[-na:, node], a[-na:, node], perm,
                                                         200 * n_envs)
    return dict(critic_loss=critic_loss, TR_loss=TR_loss, actor_loss=actor_loss)
