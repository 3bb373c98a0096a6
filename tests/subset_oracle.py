"""The exact subset-selection rules of include/rcmarl.h (rcmarl_subset_aggregate) in NumPy: MDA (minimum-diameter
averaging) and SMEA (smallest-maximum-eigenvalue averaging), with the weight w_k each gives its in-neighbours, the
margin of a selection, and an oracle agent whose hidden-layer and estimate consensus use the aggregate of the packed
messages, built on the NumPy oracle (oracle/rpbcac_oracle.py), which stays unchanged.

The distances are fp64 in either dtype, as in the kernel; the candidates are itertools.combinations of the unflagged
rows (lexicographic order); MDA's criterion is exact, SMEA's is numpy.linalg.eigvalsh of the double-centred matrix B_S
(cyclic Jacobi in the kernel); ties go to the lower rank.  The output is summed in index order in the dtype of the
messages, so the fp32 restatement is the kernel's arithmetic up to the eigen-solver."""
import itertools

import numpy as np

import attack_oracle as AT
from oracle import rpbcac_oracle as O

RULES = ("mda", "smea")


def check(H, n):
    if not (1 <= n and 0 <= H < n):
        raise ValueError(f"mda / smea do not allow H={H} with n={n}")


def flagged(X):
    """The rows that hold +-inf."""
    return np.isinf(np.asarray(X)).any(1)


def distances(X):
    """D [n, n]: fp64 squared distances of the rows (0 on the diagonal and wherever a row is flagged)."""
    X = np.asarray(X).astype(np.float64)
    n = X.shape[0]
    f = flagged(X)
    D = np.zeros((n, n))
    for k in range(n):
        for l in range(k + 1, n):
            if not (f[k] or f[l]):
                D[k, l] = D[l, k] = np.sum((X[k] - X[l]) ** 2)
    return D


def centred(D, S):
    """B_S = -1/2 J D_S J in the kernel's order: r_a = (sum_b D_ab) / s, t = (sum_a r_a) / s,
    B_ab = -0.5 (((D_ab - r_a) - r_b) + t) for a <= b, mirrored."""
    S = list(S)
    s = len(S)
    r = [sum(D[a, b] for b in S) / s for a in S]
    t = sum(r) / s
    B = np.zeros((s, s))
    for i in range(s):
        for j in range(i, s):
            B[i, j] = B[j, i] = -0.5 * (((D[S[i], S[j]] - r[i]) - r[j]) + t)
    return B


def criterion(rule, D, S):
    """c(S): 0 for a single row; MDA the largest D_ab over a < b in S; SMEA the largest eigenvalue of B_S."""
    S = list(S)
    if len(S) == 1:
        return 0.0
    if rule == "mda":
        return max(D[a, b] for a, b in itertools.combinations(S, 2))
    if rule == "smea":
        return float(np.linalg.eigvalsh(centred(D, S))[-1])
    raise ValueError(f"unknown rule {rule!r}")


def candidates(X, H):
    """(s, every s-subset of the unflagged rows in lexicographic order), s = n - max(|F|, H); no candidate when every
    row is flagged."""
    X = np.asarray(X)
    n = X.shape[0]
    f = flagged(X)
    s = n - max(int(f.sum()), H)
    U = [k for k in range(n) if not f[k]]
    return s, list(itertools.combinations(U, s)) if U else []


def _batched(rule, X, H):
    """(candidates in rank order, their criteria [C], their ordered distance submatrices [C, s, s])."""
    D = distances(X)
    s, cands = candidates(X, H)
    if not cands:
        return cands, np.zeros(0), np.zeros((0, s, s))
    idx = np.array(cands)
    Ds = D[idx[:, :, None], idx[:, None, :]]
    if s == 1:
        c = np.zeros(len(cands))
    elif rule == "mda":
        c = Ds.max((1, 2))
    elif rule == "smea":
        r = Ds.sum(2) / s
        t = r.sum(1) / s
        B = -0.5 * (((Ds - r[:, :, None]) - r[:, None, :]) + t[:, None, None])
        c = np.linalg.eigvalsh(B)[:, -1]
    else:
        raise ValueError(f"unknown rule {rule!r}")
    return cands, c, Ds


def scores(rule, X, H):
    """[(c(S), S)] over the candidates, in rank order (criterion() for every candidate, batched)."""
    cands, c, _ = _batched(rule, X, H)
    return [(float(v), S) for v, S in zip(c, cands)]


def select(rule, X, H):
    """S*: the candidate of smallest criterion, ties to the lower rank; () when every row is flagged."""
    sc = scores(rule, X, H)
    if not sc:
        return ()
    best = min(range(len(sc)), key=lambda q: (sc[q][0], q))
    return sc[best][1]


def margin(rule, X, H):
    """The relative gap (c_2 - c_1) / c_2 between the best criterion c_1 and the second-best c_2; inf with one
    candidate.  A candidate whose criterion is computed from the same numbers as c_1 ties with it in the kernel too,
    where both rules take the lower rank, so it does not count as c_2: for MDA, a candidate whose diameter is the same
    pair of rows; for SMEA, a candidate with the same ordered distance submatrix (the same rows, repeated).  Any other
    near or exact tie gives a margin near 0: rows that are equal here may differ in the kernel's inputs."""
    cands, c, Ds = _batched(rule, X, H)
    if len(cands) < 2 or Ds.shape[1] == 1:                 # one row per subset: every criterion is 0 by definition
        return np.inf
    q = min(range(len(c)), key=lambda k: (c[k], k))
    if rule == "mda":
        idx = np.array(cands)
        flat = Ds.reshape(len(cands), -1).argmax(1)          # the diameter's pair, as row indices
        pair = np.sort(np.stack([idx[np.arange(len(cands)), flat // idx.shape[1]],
                                 idx[np.arange(len(cands)), flat % idx.shape[1]]], 1), 1)
        same = (pair == pair[q]).all(1)
    else:
        same = (Ds == Ds[q]).all((1, 2))
    others = c[~same]
    if others.size == 0:
        return np.inf
    c2 = others.min()
    return (c2 - c[q]) / c2 if c2 > 0 else 0.0


def mean_of(X, sel):
    """(sum over sel, index order, of X[k]) / len(sel) in X's dtype, summed from 0."""
    X = np.asarray(X)
    dt = X.dtype.type
    s = np.zeros(X.shape[1], X.dtype)
    for k in sorted(sel):
        s = s + X[k]
    return s / dt(len(sel))


def aggregate(rule, X, H):
    """(out [P], w [n]) of MDA or SMEA over the messages X [n, P] (own = X[0]); the output in X's dtype."""
    X = np.asarray(X)
    n = X.shape[0]
    dt = X.dtype.type
    check(H, n)
    if rule not in RULES:
        raise ValueError(f"unknown rule {rule!r}")
    w = np.zeros(n, X.dtype)
    sel = select(rule, X, H)
    if not sel:                                          # every row flagged: out = own
        w[0] = dt(1)
        return X[0].copy(), w
    w[list(sel)] = dt(1) / dt(len(sel))
    return mean_of(X, sel), w


class RPBCACOracleAgent(O.RPBCACOracleAgent):
    """O.RPBCACOracleAgent whose consensus uses the MDA or SMEA aggregate of the packed messages: the hidden layers
    become the aggregate's, the estimate is phi . W3_agg + b3_agg (phi with the agent's hidden layers).  last_weights
    lists the w of every aggregation in call order, last_margins the margin() of its messages.

    Where a margin is below `gap` and kernel_w is set, the agent follows the kernel's selection: kernel_w[epoch] =
    [critic w, TR w] of the agent's job (4 aggregations per epoch: critic, TR hidden; critic, TR estimates).  Mixed or
    crafted messages can tie in exact arithmetic, where the rounding of the distances decides."""

    kernel_w = None

    def __init__(self, *args, aggregation="mda", gap=1e-6, **kw):
        super().__init__(*args, **kw)
        if aggregation not in RULES:
            raise ValueError(f"unknown rule {aggregation!r}")
        self.aggregation = aggregation
        self.gap = gap
        self.last_weights = []
        self.last_margins = []

    def _aggregate(self, w, msgs):
        X = np.stack([AT.pack(m, self.dtype) for m in msgs])
        g = margin(self.aggregation, X, self.H)
        c = len(self.last_weights)
        if g < self.gap and self.kernel_w is not None:
            keep = np.flatnonzero(self.kernel_w[c // 4][c % 2][:X.shape[0]] > 0)
            out, wt = mean_of(X, keep), np.zeros(X.shape[0], X.dtype)
            wt[keep] = 1.0 / len(keep)
        else:
            out, wt = aggregate(self.aggregation, X, self.H)
        self.last_weights.append(wt)
        self.last_margins.append(g)
        return AT.unpack(out, w)

    def _hidden(self, w, msgs):
        return self._aggregate(w, msgs)[:4] + [w[4], w[5]]

    def _estimates(self, w, x, msgs):
        agg = self._aggregate(w, msgs)
        return O.mlp_features(w, x) @ agg[4] + agg[5]


def follow_kernel(agents, runs):
    """Give each subset oracle agent the kernel's weights of epoch e from runs[e] (a Trainer whose last epoch is e)."""
    for i, ag in enumerate(agents):
        if isinstance(ag, RPBCACOracleAgent):
            ag.kernel_w = [[tr.subset_weights[2 * tr.subset_agents.index(i) + t].cpu().numpy() for t in range(2)]
                           for tr in runs]


# rounds with Byzantine agents take attack_oracle's (or adaptive_attack_oracle's) messages_hook, and rounds that mix
# nnm_oracle's or bucket_oracle's around it
update_round = AT.update_round
