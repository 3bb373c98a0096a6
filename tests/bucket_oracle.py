"""Randomized bucketing of include/rcmarl.h (rcmarl_bucket_mix) in NumPy: the Philox permutation (integer-exact, through
attack_oracle's Philox4x32-10), the buckets, the bucket means in the dtype of the messages (fp32 or fp64) with the
poisoned-row rule, and the mixing matrix M; and a messages_hook for update_round that turns the message list of every
bucketing receiver into its n_out rows, so that it composes with nnm_oracle's hook, the attack hooks and the agents of
agg_oracle, vector_oracle and dnc_oracle.  The NumPy oracle (oracle/rpbcac_oracle.py) stays unchanged."""
import numpy as np

import attack_oracle as AT

COOP = "Cooperative"
STREAM = 0x20000000                                   # bit 29 of counter word 1


def n_out(n_in, s):
    """The rows a receiver's rule reads after bucketing n_in messages at bucket size s: the own row and ceil(m / s)."""
    if n_in < 1 or s < 1:
        raise ValueError(f"bucketing needs n_in >= 1 and s >= 1, got n_in={n_in} s={s}")
    return 1 + -(-(n_in - 1) // s)


def draws(count, seed, receiver, net, round_, epoch):
    """The first `count` 32-bit draws: draw t is word t & 3 of Philox4x32-10 at counter
    (t >> 2, receiver | net << 8 | 0x20000000, round, epoch) under key (seed low word, seed high word)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if count <= 0:
        return []
    n_ctr = (count + 3) // 4
    w1 = (int(receiver) | int(net) << 8 | STREAM) & 0xFFFFFFFF
    ctr = [np.arange(n_ctr, dtype=np.uint64), np.full(n_ctr, w1, np.uint64),
           np.full(n_ctr, int(round_) & 0xFFFFFFFF, np.uint64), np.full(n_ctr, int(epoch) & 0xFFFFFFFF, np.uint64)]
    words = AT.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    return [int(words[t & 3][t >> 2]) for t in range(count)]


def permutation(n_in, seed, receiver, net, round_, epoch):
    """pi: the received slots 1 .. n_in - 1 shuffled by Fisher-Yates, i = m-1 down to 1, j = (u (i + 1)) >> 32."""
    m = n_in - 1
    pi = list(range(1, m + 1))
    u = draws(m - 1, seed, receiver, net, round_, epoch)
    for t, i in enumerate(range(m - 1, 0, -1)):
        j = (u[t] * (i + 1)) >> 32
        pi[i], pi[j] = pi[j], pi[i]
    return pi


def buckets(n_in, s, seed, receiver, net, round_, epoch):
    """The buckets of the slots, each in increasing slot order (the summation order), in bucket order."""
    n_out(n_in, s)
    pi = permutation(n_in, seed, receiver, net, round_, epoch)
    return [sorted(pi[b:b + s]) for b in range(0, len(pi), s)]


def mix(X, bks):
    """(rows [n_out, P], M [n_out, n_in]) of the messages X [n_in, P] (own = X[0]) in X's dtype: row 0 = X[0]; row
    1 + b = the fp sum from 0 of bucket b's rows in slot order, then one division by |bucket b|, or +inf throughout if
    any coordinate of that mean is not finite; M[0, 0] = 1, M[1 + b, l] = 1/|bucket b| on bucket b."""
    X = np.asarray(X)
    n, P = X.shape
    dt = X.dtype.type
    out = np.zeros((1 + len(bks), P), X.dtype)
    M = np.zeros((1 + len(bks), n), X.dtype)
    out[0] = X[0]
    M[0, 0] = 1
    with np.errstate(over="ignore", invalid="ignore"):
        for b, bk in enumerate(bks):
            s = np.zeros(P, X.dtype)
            for l in bk:
                s = s + X[l]
            mean = s / dt(len(bk))
            out[1 + b] = mean if np.isfinite(mean).all() else np.inf
            M[1 + b, bk] = dt(1) / dt(len(bk))
    return out, M


def bucket_mix(X, s, seed, receiver, net, round_, epoch):
    """mix(X, buckets(...)) of one job."""
    return mix(X, buckets(np.asarray(X).shape[0], s, seed, receiver, net, round_, epoch))


def bucketing_hook(labels, in_nodes, mixing, seed, round_, inner=None, log=None):
    """messages_hook of update_round: the critic and TR message lists of every cooperative receiver j whose mixing[j]
    is ("bucket", s) (inner(epoch, ...)'s lists if inner is given, else those of in_nodes[j]) become its n_out rows,
    drawn as the Trainer draws them (receiver j, net 0 critic / 1 TR, the round and the epoch).  Receivers with any
    other entry keep inner's lists, so an nnm hook goes inside or outside this one.  log (a dict), when given, receives
    per bucketing receiver one entry per epoch: [(M, X) of the critic, ... of the TR net]."""
    coop = [j for j, l in enumerate(labels) if l == COOP]

    def hook(epoch, critic_msgs, TR_msgs):
        if inner is None:
            per_c = {j: [critic_msgs[i] for i in in_nodes[j]] for j in coop}
            per_t = {j: [TR_msgs[i] for i in in_nodes[j]] for j in coop}
        else:
            per_c, per_t = (dict(x) for x in inner(epoch, critic_msgs, TR_msgs))
        for j in coop:
            if not (isinstance(mixing[j], tuple) and mixing[j][0] == "bucket"):
                continue
            entry = []
            for net, per in enumerate((per_c, per_t)):
                msgs = per[j]
                X = np.stack([AT.pack(m, np.asarray(msgs[0][0]).dtype) for m in msgs])
                Y, M = bucket_mix(X, mixing[j][1], seed, j, net, round_, epoch)
                per[j] = [AT.unpack(Y[k], msgs[0]) for k in range(Y.shape[0])]
                entry.append((M, X))
            if log is not None:
                log.setdefault(j, []).append(entry)
        return per_c, per_t
    return hook


# rounds that bucket take bucketing_hook (around an attack hook where there are Byzantine agents)
update_round = AT.update_round
