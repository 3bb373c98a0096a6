"""The resilient aggregation rules of include/rcmarl.h (rcmarl_agg_rule) on top of the NumPy oracle
(oracle/rpbcac_oracle.py), in the oracle's dtype (fp32 or fp64).  "clip" is the oracle's own resilient_aggregation, so
every clip result is the one the reference comparisons already pin; "trim" and "wmsr" keep a tie-broken rank range
and add the kept values in index order, as the kernels do."""
import numpy as np

from oracle import rpbcac_oracle as O

RULES = ("clip", "trim", "wmsr")


def keep_mask(values, H, rule):
    """Boolean mask of the values "trim" / "wmsr" keep, over axis 0 (own = values[0]).
    rank(k) = #{m : v[m] < v[k] or (v[m] == v[k] and m < k)} is the position of k in a stable sort."""
    v = np.asarray(values)
    n = v.shape[0]
    order = np.argsort(v, axis=0, kind="stable")
    rank = np.empty_like(order)
    np.put_along_axis(rank, order, np.broadcast_to(np.arange(n).reshape((n,) + (1,) * (v.ndim - 1)), v.shape), axis=0)
    if rule == "trim":
        if not 0 <= 2 * H < n:
            raise ValueError(f"trim needs 0 <= 2H < n (H={H}, n={n})")
        lo, hi = H, n - H - 1
    elif rule == "wmsr":
        if not 0 <= H < n:
            raise ValueError(f"wmsr needs 0 <= H < n (H={H}, n={n})")
        above, below = (v > v[0]).sum(0), (v < v[0]).sum(0)
        lo, hi = np.minimum(H, below), n - 1 - np.minimum(H, above)
    else:
        raise ValueError(f"unknown rule {rule!r}")
    return (rank >= lo) & (rank <= hi)


def resilient_aggregation(values, H, rule="clip"):
    """Aggregate over axis 0 (own = values[0]) in values' dtype."""
    if rule == "clip":
        return O.resilient_aggregation(values, H)
    v = np.asarray(values)
    keep = keep_mask(v, H, rule)
    s = np.zeros(v.shape[1:], v.dtype)
    for k in range(v.shape[0]):                          # index order; a dropped value never enters the sum
        s = s + np.where(keep[k], v[k], v.dtype.type(0))
    return (s / keep.sum(0).astype(v.dtype)).astype(v.dtype)


class RPBCACOracleAgent(O.RPBCACOracleAgent):
    """O.RPBCACOracleAgent whose hidden-layer and estimate consensus use `aggregation`."""

    def __init__(self, *args, aggregation="clip", **kw):
        super().__init__(*args, **kw)
        if aggregation not in RULES:
            raise ValueError(f"unknown rule {aggregation!r}")
        self.aggregation = aggregation

    def _hidden(self, w, msgs):
        agg = [resilient_aggregation(np.stack([np.asarray(m[k], self.dtype) for m in msgs]), self.H, self.aggregation)
               for k in range(6)]
        return agg[:4] + [w[4], w[5]]

    def _estimates(self, w, x, msgs):
        phi = O.mlp_features(w, x)
        ests = np.stack([phi @ np.asarray(m[4], self.dtype) + np.asarray(m[5], self.dtype) for m in msgs])
        return resilient_aggregation(ests, self.H, self.aggregation)


# the update round calls the agents' methods, so each cooperative agent's rule is the one it was built with
update_round = O.update_round
