"""Nearest-neighbour mixing of include/rcmarl.h (rcmarl_nnm_mix) in NumPy, in the dtype of the messages (fp32 or fp64),
with its mixing matrix M; and a messages_hook for update_round that mixes the messages each mixing receiver hears
before its own rule runs, so that it composes with the agents of agg_oracle, vector_oracle and dnc_oracle and with the
attack hooks.  The NumPy oracle (oracle/rpbcac_oracle.py) stays unchanged.

Distances are vector_oracle's: a squared distance that is not finite or exceeds the fp32 range counts as +inf in
either dtype, as in the kernel, whose distances are fp32."""
import numpy as np

import attack_oracle as AT
import vector_oracle as VO

COOP = "Cooperative"


def check(H, n):
    if not (1 <= n and 0 <= H < n):
        raise ValueError(f"nnm does not allow H={H} with n={n}")


def order(D, k):
    """The rows l ordered by (D_kl, l != k, l) for row k, with D_kk = 0."""
    n = D.shape[0]
    d = [0.0 if l == k else D[k, l] for l in range(n)]
    return sorted(range(n), key=lambda l: (d[l], l != k, l))


def selections(X, H):
    """N_k for every k: the first n - H of order(D, k), less every l at distance +inf (index order)."""
    X = np.asarray(X)
    n = X.shape[0]
    check(H, n)
    D = VO.pairwise(X)
    return [sorted(l for l in order(D, k)[:n - H] if l == k or np.isfinite(D[k, l])) for k in range(n)]


def mix(X, H, sel=None):
    """(mixed [n, P], M [n, n]) of the messages X [n, P] (own = X[0]) in X's dtype: mixed_k = the sum of the rows of
    N_k in index order, then one division by |N_k|; M_kl = 1/|N_k| on N_k.  sel: the N_k to use instead of
    selections(X, H)."""
    X = np.asarray(X)
    n, P = X.shape
    dt = X.dtype.type
    out = np.zeros((n, P), X.dtype)
    M = np.zeros((n, n), X.dtype)
    for k, sel in enumerate(selections(X, H) if sel is None else sel):
        s = np.zeros(P, X.dtype)
        for l in sel:
            s = s + X[l]
        out[k] = s / dt(len(sel))
        M[k, sel] = dt(1) / dt(len(sel))
    return out, M


def margin(X, H):
    """The smallest relative gap over the rows k between the last distance a inside the first n - H of order(D, k) and
    the first b outside (both to rows other than k): (b - a) / b, inf where there is no such boundary (H = 0,
    H = n - 1) or b = +inf.  Where the rows on both sides are identical (a repeated in-node), the tie is exact in any
    precision and broken by index in both, so the gap is taken from a to the nearest distance of a row that differs
    from them."""
    X = np.asarray(X)
    n = X.shape[0]
    check(H, n)
    if H == 0 or H == n - 1:
        return np.inf
    D = VO.pairwise(X).astype(np.float64)
    worst = np.inf
    for k in range(n):
        o = order(D, k)
        la, lb = o[n - H - 1], o[n - H]
        a, b = D[k, la], D[k, lb]
        if np.isinf(b):
            continue
        if np.array_equal(X[la], X[lb]):
            g = min([abs(D[k, l] - a) / max(D[k, l], a) for l in range(n)
                     if l != k and not np.array_equal(X[l], X[la])], default=np.inf)
        else:
            g = (b - a) / b if b > 0 else 0.0
        worst = min(worst, g)
    return worst


def clear(X, H, gap=1e-4):
    """True where the kernel's fp32 selections must equal the oracle's: every boundary gap above `gap`."""
    return margin(X, H) > gap


def mixing_hook(labels, in_nodes, mixing, H, inner=None, log=None, kernel_M=None):
    """messages_hook of update_round: the critic and TR message lists of every cooperative receiver j with mixing[j]
    (inner(epoch, ...)'s lists if inner is given, else those of in_nodes[j]) become their n mixed messages, own =
    mixed row 0; the receiver's rule then runs on them.  log (a dict), when given, receives per mixing receiver one
    entry per epoch: [(M, X, clear) of the critic, ... of the TR net], X the packed messages before mixing.
    kernel_M[epoch][j] ([2, n, n], e.g. Trainer.mixing_matrices()), when given, supplies the selections where they
    are not clear(X, H): there a near tie may fall either way in fp32, and the oracle follows the kernel's pick."""
    coop = [j for j, l in enumerate(labels) if l == COOP]

    def hook(epoch, critic_msgs, TR_msgs):
        if inner is None:
            per_c = {j: [critic_msgs[i] for i in in_nodes[j]] for j in coop}
            per_t = {j: [TR_msgs[i] for i in in_nodes[j]] for j in coop}
        else:
            per_c, per_t = (dict(x) for x in inner(epoch, critic_msgs, TR_msgs))
        for j in coop:
            if mixing[j] is None:
                continue
            entry = []
            for per in (per_c, per_t):
                msgs = per[j]
                X = np.stack([AT.pack(m, np.asarray(msgs[0][0]).dtype) for m in msgs])
                ok = clear(X, H[j])
                sel = None
                if not ok and kernel_M is not None and j in kernel_M.get(epoch, {}):
                    sel = [list(np.flatnonzero(row > 0)) for row in kernel_M[epoch][j][len(entry)]]
                Y, M = mix(X, H[j], sel)
                per[j] = [AT.unpack(Y[k], msgs[0]) for k in range(len(msgs))]
                entry.append((M, X, ok))
            if log is not None:
                log.setdefault(j, []).append(entry)
        return per_c, per_t
    return hook


# rounds that mix take mixing_hook (around an attack hook where there are Byzantine agents)
update_round = AT.update_round
