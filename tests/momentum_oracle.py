"""Per-neighbour momentum of include/rcmarl.h (rcmarl_momentum_mix) in NumPy: one step of the state M and the momentum
rows in the dtype of the messages (fp32: every operation rounded on its own, as NumPy float32 arithmetic does, so it
is the kernel's arithmetic bit for bit), and a messages_hook for update_round that turns the message list of every
receiver with momentum into its momentum rows against the receiver's own nets, carrying M over between epochs and
rounds.  It composes with the attack hooks and the agents of agg_oracle, vector_oracle, dnc_oracle and subset_oracle.
The NumPy oracle (oracle/rpbcac_oracle.py) stays unchanged."""
import numpy as np

import attack_oracle as AT

COOP = "Cooperative"


def step(X, c, M, beta, first):
    """(rows [n, P], new M [n, P]) of the messages X [n, P] (own = X[0]), the reference c [P] and the state M [n, P] (not
    read when first) in X's dtype: u = X - c; M' = u if first or where M is finite and u is not, M where M is +-inf,
    beta M + (1 - beta) u elsewhere; rows = c + M'."""
    X = np.asarray(X)
    dt = X.dtype.type
    c = np.asarray(c, X.dtype)
    with np.errstate(over="ignore", invalid="ignore"):
        u = X - c
        if first:
            new = u.copy()
        else:
            M = np.asarray(M, X.dtype)
            b = dt(beta)
            ema = b * M + (dt(1) - b) * u
            new = np.where(np.isinf(M), M, np.where(np.isfinite(u), ema, u))
        return c + new, new


class MomentumHook:
    """messages_hook of update_round: the critic and TR message lists of every cooperative receiver j with
    momentum[j] not None (inner(epoch, ...)'s lists if inner is given, else those of in_nodes[j]) become its momentum
    rows against agents[j]'s critic and TR nets as they stand when the hook runs (after Phase I, before any consensus:
    the nets of the previous consensus step).  One call is one epoch; M[(j, net)] carries over between calls and
    rounds, and a receiver's first call is its first step.  log (a dict), when given, receives per receiver one entry
    per epoch: [(X, c, rows, M) of the critic, ... of the TR net]."""

    def __init__(self, agents, labels, in_nodes, momentum, inner=None, log=None):
        self.agents, self.labels, self.in_nodes, self.momentum = agents, labels, in_nodes, momentum
        self.inner, self.log = inner, log
        self.M = {}

    def __call__(self, epoch, critic_msgs, TR_msgs):
        coop = [j for j, l in enumerate(self.labels) if l == COOP]
        if self.inner is None:
            per_c = {j: [critic_msgs[i] for i in self.in_nodes[j]] for j in coop}
            per_t = {j: [TR_msgs[i] for i in self.in_nodes[j]] for j in coop}
        else:
            per_c, per_t = (dict(x) for x in self.inner(epoch, critic_msgs, TR_msgs))
        for j in coop:
            if self.momentum[j] is None:
                continue
            entry = []
            for net, per in enumerate((per_c, per_t)):
                msgs = per[j]
                dt = np.asarray(msgs[0][0]).dtype
                X = np.stack([AT.pack(m, dt) for m in msgs])
                c = AT.pack(self.agents[j].get_parameters()[1 + net], dt)
                first = (j, net) not in self.M
                rows, self.M[(j, net)] = step(X, c, self.M.get((j, net)), self.momentum[j], first)
                per[j] = [AT.unpack(rows[k], msgs[0]) for k in range(rows.shape[0])]
                entry.append((X, c, rows, self.M[(j, net)]))
            if self.log is not None:
                self.log.setdefault(j, []).append(entry)
        return per_c, per_t


# rounds with momentum take MomentumHook (around an attack hook where there are Byzantine agents)
update_round = AT.update_round
