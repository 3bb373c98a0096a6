"""The distance-based resilient aggregation rules of include/rcmarl.h (rcmarl_vector_rule: krum, mkrum, scclip, gmed) in
NumPy, in the dtype of the messages (fp32 or fp64), with the weight w_k each rule gives each in-neighbour; and an oracle
agent whose hidden-layer and estimate consensus use the aggregate of the packed messages, built on the NumPy oracle
(oracle/rpbcac_oracle.py), which stays unchanged.

The kernel's distances are fp32, so here a squared distance that is not finite or exceeds the fp32 range counts as +inf
in either dtype: a message of 1e30 is at an infinite distance in both; and a term that underflows in fp32 is 0 in both."""
import numpy as np

import agg_oracle as AO
import attack_oracle as AT
from oracle import rpbcac_oracle as O

RULES = ("krum", "mkrum", "scclip", "gmed")
GMED_ITERS, GMED_NU = 8, 1e-6
F32_MAX = float(np.finfo(np.float32).max)
F32_HALF_TINY = 2.0 ** -150                          # half the smallest fp32 subnormal: rounds to 0


def sqdist(a, b):
    """sum_p (a_p - b_p)^2 in a's dtype; +inf where not finite or beyond the fp32 range.  A term below half the
    smallest fp32 subnormal is 0, as the kernel's fp32 product rounds it: in fp64 too, rows that differ by less than
    about 1e-23 per coordinate are at distance 0."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = np.asarray(a) - np.asarray(b)
        t = d * d
        s = np.where(t <= F32_HALF_TINY, t.dtype.type(0), t).sum(-1)
    return s if np.isfinite(s) and s <= F32_MAX else s.dtype.type(np.inf)


def pairwise(X):
    n = X.shape[0]
    D = np.zeros((n, n), X.dtype)
    for k in range(n):
        for l in range(k + 1, n):
            D[k, l] = D[l, k] = sqdist(X[k], X[l])
    return D


def krum_scores(X, H):
    """score_k = the n - H - 2 smallest D_kl over l != k, added in ascending order."""
    n = X.shape[0]
    D = pairwise(X)
    out = np.zeros(n, X.dtype)
    for k in range(n):
        s = X.dtype.type(0)
        for v in np.sort(np.delete(D[k], k))[:n - H - 2]:
            s = s + v
        out[k] = s
    return out


def check(rule, H, n):
    if rule not in RULES:
        raise ValueError(f"unknown rule {rule!r}")
    if not 0 <= H < n or (rule in ("krum", "mkrum") and n < H + 3):
        raise ValueError(f"{rule} does not allow H={H} with n={n}")


def aggregate(X, H, rule):
    """(out [P], w [n]) of `rule` over the messages X [n, P] (own = X[0]) in X's dtype."""
    X = np.asarray(X)
    n, P = X.shape
    dt = X.dtype.type
    check(rule, H, n)
    if rule in ("krum", "mkrum"):
        m = 1 if rule == "krum" else n - H
        sel = sorted(np.argsort(krum_scores(X, H), kind="stable")[:m])       # ties to the lower index
        w = np.zeros(n, X.dtype)
        w[sel] = dt(1) / dt(m)
        s = np.zeros(P, X.dtype)
        for k in sel:
            s = s + X[k]
        return s / dt(m), w
    if rule == "scclip":
        d = np.array([np.sqrt(sqdist(X[k], X[0])) for k in range(1, n)], X.dtype)
        tau = dt(0) if H >= n - 1 else -np.sort(-d)[H]                       # the (H+1)-th largest
        with np.errstate(divide="ignore", invalid="ignore"):
            c = np.where(~np.isfinite(d), dt(0), np.where(d <= tau, dt(1), tau / d)).astype(X.dtype)
        s = np.zeros(P, X.dtype)
        for k in range(1, n):
            if c[k - 1] != 0:
                s = s + c[k - 1] * (X[k] - X[0])
        w = np.concatenate([[dt(0)], c / dt(n)]).astype(X.dtype)
        w[0] = dt(1) - w[1:].sum(dtype=X.dtype)
        return X[0] + s / dt(n), w
    z = AO.resilient_aggregation(X, (n - 1) // 2, "trim")                   # the coordinate-wise median
    for _ in range(GMED_ITERS):
        d = np.array([np.sqrt(sqdist(X[k], z)) for k in range(n)], X.dtype)
        beta = np.where(np.isfinite(d), dt(1) / np.maximum(d, dt(GMED_NU)), dt(0)).astype(X.dtype)
        S = dt(0)
        for b in beta:
            S = S + b
        if S == 0:                                                           # no finite distance: out = own
            beta[0], S = dt(1), dt(1)
        s = np.zeros(P, X.dtype)
        for k in range(n):
            if beta[k] != 0:
                s = s + beta[k] * X[k]
        z = s / S
    return z, beta / S


class RPBCACOracleAgent(O.RPBCACOracleAgent):
    """O.RPBCACOracleAgent whose consensus uses the aggregate of a distance-based rule over the packed messages: the
    hidden layers become the aggregate's, the estimate is phi . W3_agg + b3_agg (phi with the agent's hidden layers).
    last_weights lists the w of every aggregation in call order."""

    def __init__(self, *args, aggregation="krum", **kw):
        super().__init__(*args, **kw)
        if aggregation not in RULES:
            raise ValueError(f"unknown rule {aggregation!r}")
        self.aggregation = aggregation
        self.last_weights = []

    def _aggregate(self, w, msgs):
        out, wt = aggregate(np.stack([AT.pack(m, self.dtype) for m in msgs]), self.H, self.aggregation)
        self.last_weights.append(wt)
        return AT.unpack(out, w)

    def _hidden(self, w, msgs):
        return self._aggregate(w, msgs)[:4] + [w[4], w[5]]

    def _estimates(self, w, x, msgs):
        agg = self._aggregate(w, msgs)
        return O.mlp_features(w, x) @ agg[4] + agg[5]


# rounds with Byzantine agents take attack_oracle's messages_hook; the agents' methods carry each agent's rule
update_round = AT.update_round
