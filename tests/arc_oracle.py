"""Adaptive robust clipping of include/rcmarl.h (rcmarl_arc_clip) in NumPy: the distances d_k, k_clip, tau and the
factors c in fp64; the rows given c in the dtype of the messages (fp32: every operation rounded on its own, as NumPy
float32 arithmetic does, so it is the kernel's arithmetic bit for bit); and a messages_hook for update_round that
clips the message list of every receiver that clips.  It composes with MomentumHook (inside it), the nnm and bucketing
hooks (around it) and the attack hooks, in the trainer's order.  The NumPy oracle (oracle/rpbcac_oracle.py) stays
unchanged."""
import numpy as np

import attack_oracle as AT

COOP = "Cooperative"


def k_clip(H, n):
    """How many of n messages ARC may clip at H: floor(2 (H / n) (n - H)) = (2 H (n - H)) // n."""
    return (2 * H * (n - H)) // n


def distances(X):
    """d_k = ||x_k - x_0|| for k >= 1 in fp64 (d_0 = 0); a distance that is not finite is +inf, and so is one whose
    square lies beyond the fp32 range, where the kernel's fp32 sum overflows (a 1e30 coordinate)."""
    X = np.asarray(X, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        sq = ((X - X[0]) ** 2).sum(1)
    sq[~(sq <= float(np.finfo(np.float32).max))] = np.inf
    d = np.sqrt(sq)
    d[0] = 0.0
    return d


def factors(X, H, d=None):
    """(c [n], tau) of the messages X [n, P] (own = X[0]) at H, in fp64: tau the (k_clip + 1)-th largest d_k, k >= 1
    (0 if k_clip >= n - 1); c_0 = 1, c_k = 0 where d_k is +inf, 1 where d_k <= tau, tau / d_k elsewhere.  d, when given,
    replaces the fp64 distances (e.g. the kernel's own, to follow its ranking at near ties)."""
    n = len(X)
    d = distances(X) if d is None else np.asarray(d, np.float64)
    kc = k_clip(H, n)
    tau = 0.0 if kc >= n - 1 else np.sort(d[1:])[::-1][kc]
    c = np.ones(n)
    with np.errstate(invalid="ignore", divide="ignore"):
        for k in range(1, n):
            c[k] = 0.0 if not np.isfinite(d[k]) else (1.0 if d[k] <= tau else tau / d[k])
    return c, tau


def rows(X, c):
    """The clipped rows of the messages X [n, P] given c [n], in X's dtype: x_k where c_k = 1, x_0 where c_k = 0,
    x_0 + c_k (x_k - x_0) elsewhere (fp32: each operation rounded on its own)."""
    X = np.asarray(X)
    dt = X.dtype.type
    out = X.copy()
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(1, len(X)):
            ck = dt(c[k])
            if ck == 0:
                out[k] = X[0]
            elif ck != 1:
                out[k] = X[0] + ck * (X[k] - X[0])
    return out


def clip(X, H):
    """(rows, c, tau) of ARC in X's dtype with the factors of `factors`: fp64 inputs give the fp64 oracle."""
    c, tau = factors(X, H)
    return rows(X, c), c, tau


class ArcHook:
    """messages_hook of update_round: the critic and TR message lists of every cooperative receiver j with clipping[j]
    not None (inner(epoch, ...)'s lists if inner is given, else those of in_nodes[j]; inner may be a MomentumHook) become
    its n clipped rows at H[j].  log (a dict), when given, receives per receiver one entry per epoch: [(X, c, tau) of the
    critic, ... of the TR net]."""

    def __init__(self, labels, in_nodes, clipping, H, inner=None, log=None):
        self.labels, self.in_nodes, self.clipping, self.H = labels, in_nodes, clipping, H
        self.inner, self.log = inner, log

    def __call__(self, epoch, critic_msgs, TR_msgs):
        coop = [j for j, l in enumerate(self.labels) if l == COOP]
        if self.inner is None:
            per_c = {j: [critic_msgs[i] for i in self.in_nodes[j]] for j in coop}
            per_t = {j: [TR_msgs[i] for i in self.in_nodes[j]] for j in coop}
        else:
            per_c, per_t = (dict(x) for x in self.inner(epoch, critic_msgs, TR_msgs))
        for j in coop:
            if self.clipping[j] is None:
                continue
            entry = []
            for per in (per_c, per_t):
                msgs = per[j]
                X = np.stack([AT.pack(m, np.asarray(msgs[0][0]).dtype) for m in msgs])
                Y, c, tau = clip(X, self.H[j])
                per[j] = [AT.unpack(Y[k], msgs[0]) for k in range(len(msgs))]
                entry.append((X, c, tau))
            if self.log is not None:
                self.log.setdefault(j, []).append(entry)
        return per_c, per_t


# rounds that clip take ArcHook (around a momentum or an attack hook, inside a mixing hook)
update_round = AT.update_round
