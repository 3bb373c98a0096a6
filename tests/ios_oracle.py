"""The iterative outlier scissor (IOS) of include/rcmarl.h (rcmarl_ios_aggregate) in NumPy, with the weight w_k it gives
each in-neighbour, the margin of its removals, and an oracle agent whose hidden-layer and estimate consensus use the IOS
aggregate of the packed messages, built on the NumPy oracle (oracle/rpbcac_oracle.py), which stays unchanged.

The centre and the distances are fp64 in either dtype, as in the kernel (summed in another order there); the output
is summed in index order in the dtype of the messages, so the fp32 restatement is the kernel's output arithmetic."""
import numpy as np

import attack_oracle as AT
from oracle import rpbcac_oracle as O


def check(H, n):
    if not (1 <= n and 0 <= H < n):
        raise ValueError(f"ios does not allow H={H} with n={n}")


def flagged(X):
    """The rows that hold +-inf."""
    return np.isinf(np.asarray(X)).any(1)


def centre(X, U):
    """c = (sum over U, index order, of (double)x_k) / |U| in fp64."""
    X = np.asarray(X)
    c = np.zeros(X.shape[1])
    for k in U:
        c = c + X[k].astype(np.float64)
    return c / len(U)


def distances(X, U):
    """{k: d_k = sum_p ((double)x_k,p - c_p)^2} over U, with c = centre(X, U)."""
    X = np.asarray(X)
    c = centre(X, U)
    return {k: float(np.sum((X[k].astype(np.float64) - c) ** 2)) for k in U}


def steps(X, H):
    """[(U before the step, d over U, removed row)] of every iteration: max(0, H - |F|) of them (none when every row is
    flagged); equal d remove the higher index first."""
    X = np.asarray(X)
    f = flagged(X)
    U = [k for k in range(X.shape[0]) if not f[k]]
    out = []
    if not U:
        return out
    for _ in range(max(0, H - int(f.sum()))):
        d = distances(X, U)
        top = max(U, key=lambda k: (d[k], k))
        out.append((list(U), d, top))
        U = [k for k in U if k != top]
    return out


def kept(X, H):
    """I: the rows left, in index order; () when every row is flagged."""
    X = np.asarray(X)
    f = flagged(X)
    gone = {top for _, _, top in steps(X, H)}
    return tuple(k for k in range(X.shape[0]) if not f[k] and k not in gone)


def margin(X, H):
    """The smallest relative gap (d_1 - d_2) / d_1 between the largest distance and the next over the iterations with
    three rows or more; inf without one.  A row equal to the removed one (a repeated in-node) has the same d in the
    kernel too, where both break the tie to the higher index, so it does not count as d_2; nor does the step from two
    rows, which lie equally far from their mean (include/rcmarl.h: with exact fp64 sums both sides compute equal d)."""
    X = np.asarray(X)
    g = np.inf
    for U, d, top in steps(X, H):
        if len(U) < 3:
            continue
        others = [d[k] for k in U if not np.array_equal(X[k], X[top])]
        if not others:
            continue
        d2 = max(others)
        g = min(g, (d[top] - d2) / d[top] if d[top] > 0 else 0.0)
    return g


def mean_of(X, sel):
    """(sum over sel, index order, of X[k]) / len(sel) in X's dtype, summed from 0."""
    X = np.asarray(X)
    dt = X.dtype.type
    s = np.zeros(X.shape[1], X.dtype)
    for k in sorted(sel):
        s = s + X[k]
    return s / dt(len(sel))


def aggregate(X, H):
    """(out [P], w [n]) of IOS over the messages X [n, P] (own = X[0]); the output in X's dtype."""
    X = np.asarray(X)
    n = X.shape[0]
    dt = X.dtype.type
    check(H, n)
    w = np.zeros(n, X.dtype)
    sel = kept(X, H)
    if not sel:                                          # every row flagged: out = own
        w[0] = dt(1)
        return X[0].copy(), w
    w[list(sel)] = dt(1) / dt(len(sel))
    return mean_of(X, sel), w


class RPBCACOracleAgent(O.RPBCACOracleAgent):
    """O.RPBCACOracleAgent whose consensus uses the IOS aggregate of the packed messages: the hidden layers become the
    aggregate's, the estimate is phi . W3_agg + b3_agg (phi with the agent's hidden layers).  last_weights lists the w of
    every aggregation in call order, last_margins the margin() of its messages.

    Where a margin is below `gap` and kernel_w is set, the agent follows the kernel's selection: kernel_w[epoch] =
    [critic w, TR w] of the agent's job (4 aggregations per epoch: critic, TR hidden; critic, TR estimates).  Mixed,
    clipped or crafted messages can tie in exact arithmetic, where the rounding of the distances decides."""

    kernel_w = None

    def __init__(self, *args, aggregation="ios", gap=1e-6, **kw):
        super().__init__(*args, **kw)
        if aggregation != "ios":
            raise ValueError(f"unknown rule {aggregation!r}")
        self.aggregation = aggregation
        self.gap = gap
        self.last_weights = []
        self.last_margins = []

    def _aggregate(self, w, msgs):
        X = np.stack([AT.pack(m, self.dtype) for m in msgs])
        g = margin(X, self.H)
        c = len(self.last_weights)
        if g < self.gap and self.kernel_w is not None:
            keep = np.flatnonzero(self.kernel_w[c // 4][c % 2][:X.shape[0]] > 0)
            out, wt = mean_of(X, keep), np.zeros(X.shape[0], X.dtype)
            wt[keep] = 1.0 / len(keep)
        else:
            out, wt = aggregate(X, self.H)
        self.last_weights.append(wt)
        self.last_margins.append(g)
        return AT.unpack(out, w)

    def _hidden(self, w, msgs):
        return self._aggregate(w, msgs)[:4] + [w[4], w[5]]

    def _estimates(self, w, x, msgs):
        agg = self._aggregate(w, msgs)
        return O.mlp_features(w, x) @ agg[4] + agg[5]


def follow_kernel(agents, runs):
    """Give each IOS oracle agent the kernel's weights of epoch e from runs[e] (a Trainer whose last epoch is e)."""
    for i, ag in enumerate(agents):
        if isinstance(ag, RPBCACOracleAgent):
            ag.kernel_w = [[tr.ios_weights[2 * tr.ios_agents.index(i) + t].cpu().numpy() for t in range(2)]
                           for tr in runs]


# rounds with Byzantine agents take attack_oracle's (or adaptive_attack_oracle's) messages_hook, and rounds that mix,
# clip or keep momentum the hooks of nnm_oracle, bucket_oracle, arc_oracle and momentum_oracle around it
update_round = AT.update_round
