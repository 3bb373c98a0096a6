"""The divide-and-conquer (DnC) rule of include/rcmarl.h (rcmarl_dnc_aggregate) in NumPy, with the weight w_k it gives
each in-neighbour; and an oracle agent whose hidden-layer and estimate consensus use the DnC aggregate of the packed
messages, built on the NumPy oracle (oracle/rpbcac_oracle.py), which stays unchanged.

The centring, the Gram matrix and its top eigenpair are fp64 in either dtype, as in the kernel (numpy.linalg.eigh here,
cyclic Jacobi there); the output is summed in the dtype of the messages, so the fp32 restatement is the kernel's
arithmetic up to the eigen-solver and the fp64 one is the exact rule."""
import numpy as np

import attack_oracle as AT
from oracle import rpbcac_oracle as O


def check(H, n):
    if not (1 <= n and 0 <= H < n):
        raise ValueError(f"dnc does not allow H={H} with n={n}")


def flagged(X):
    """The rows that hold +-inf."""
    return np.isinf(np.asarray(X)).any(1)


def spectrum(X):
    """(eigenvalues ascending, eigenvectors) of the fp64 Gram matrix of the centred unflagged rows (index order)."""
    X = np.asarray(X)
    U = X[~flagged(X)].astype(np.float64)
    mu = np.zeros(X.shape[1])
    for row in U:                                        # summed in index order
        mu = mu + row
    C = U - mu / U.shape[0]
    return np.linalg.eigh(C @ C.T)


def scores(X):
    """score_k = lambda u_k^2 for the unflagged rows (u in their index order), +inf for the flagged ones; fp64."""
    X = np.asarray(X)
    f = flagged(X)
    out = np.full(X.shape[0], np.inf)
    if (~f).any():
        lam, V = spectrum(X)
        out[~f] = lam[-1] * V[:, -1] ** 2
    return out


def removed(X, H):
    """The removed rows: every flagged row, then the H - |F| highest scores (equal scores: the higher index first)."""
    sc = scores(X)
    n_rm = max(int(flagged(X).sum()), H)
    return sorted(sorted(range(len(sc)), key=lambda k: (-sc[k], -k))[:n_rm])


def margins(X, H):
    """(relative eigengap (lambda_1 - lambda_2) / lambda_1, relative score gap at the removal boundary) of the unflagged
    rows; inf where there is no second eigenvalue or no boundary inside them."""
    f = flagged(X)
    m = int((~f).sum())
    if m == 0:
        return np.inf, np.inf
    lam, _ = spectrum(X)
    eig = np.inf if m == 1 else ((lam[-1] - lam[-2]) / lam[-1] if lam[-1] > 0 else 0.0)
    h = H - int(f.sum())
    if h <= 0 or h >= m:
        return eig, np.inf
    s = np.sort(scores(X)[~f])[::-1]
    return eig, (s[h - 1] - s[h]) / s[h - 1] if s[h - 1] > 0 else 0.0


def aggregate(X, H):
    """(out [P], w [n]) of DnC over the messages X [n, P] (own = X[0]); the output in X's dtype."""
    X = np.asarray(X)
    n, P = X.shape
    dt = X.dtype.type
    check(H, n)
    w = np.zeros(n, X.dtype)
    if flagged(X).all():                                 # no unflagged row: out = own
        w[0] = dt(1)
        return X[0].copy(), w
    gone = set(removed(X, H))
    keep = [k for k in range(n) if k not in gone]
    w[keep] = dt(1) / dt(len(keep))
    s = np.zeros(P, X.dtype)
    for k in keep:
        s = s + X[k]
    return s / dt(len(keep)), w


class RPBCACOracleAgent(O.RPBCACOracleAgent):
    """O.RPBCACOracleAgent whose consensus uses the DnC aggregate of the packed messages: the hidden layers become the
    aggregate's, the estimate is phi . W3_agg + b3_agg (phi with the agent's hidden layers).  last_weights lists the w of
    every aggregation in call order, last_margins the margins() of its messages."""

    def __init__(self, *args, aggregation="dnc", **kw):
        super().__init__(*args, **kw)
        if aggregation != "dnc":
            raise ValueError(f"unknown rule {aggregation!r}")
        self.aggregation = aggregation
        self.last_weights = []
        self.last_margins = []

    def _aggregate(self, w, msgs):
        X = np.stack([AT.pack(m, self.dtype) for m in msgs])
        out, wt = aggregate(X, self.H)
        self.last_weights.append(wt)
        self.last_margins.append(margins(X, self.H))
        return AT.unpack(out, w)

    def _hidden(self, w, msgs):
        return self._aggregate(w, msgs)[:4] + [w[4], w[5]]

    def _estimates(self, w, x, msgs):
        agg = self._aggregate(w, msgs)
        return O.mlp_features(w, x) @ agg[4] + agg[5]


# rounds with Byzantine agents take attack_oracle's (or adaptive_attack_oracle's) messages_hook
update_round = AT.update_round
