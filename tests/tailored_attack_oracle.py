"""The rule-aware Byzantine messages of include/rcmarl.h (rcmarl_tailored_attack) in NumPy, in the dtype of the messages
(fp32 or fp64), built on adaptive_attack_oracle (mu, d, gamma_mm), agg_oracle (the coordinate-wise rules) and
vector_oracle (the distance-based rules): craft() returns the message, gamma_i* and the whole objective vector O; and a
messages hook for attack_oracle.update_round that crafts these next to the attacks of adaptive_attack_oracle.make_hook.

As in the kernel, an objective that is not finite or exceeds the fp32 range counts as -inf in either dtype."""
import numpy as np

import adaptive_attack_oracle as AA
import agg_oracle as AO
import attack_oracle as AT
import vector_oracle as VO

STEPS = 32                                               # RCMARL_TAILORED_STEPS
ATTACKS = tuple(f"tailored_{d}" for d in AA.DEVS)
COORD_RULES = ("clip", "trim", "wmsr")
RULES = COORD_RULES + VO.RULES
F32_MAX = float(np.finfo(np.float32).max)


def rule_output(X, rule, H):
    """R_j(X) of the receiver's rule over the slot messages X [n_in, P] (own = X[0])."""
    if rule in VO.RULES:
        return VO.aggregate(X, H, rule)[0]
    if rule not in COORD_RULES:
        raise ValueError(f"unknown rule {rule!r}")
    return AO.resilient_aggregation(X, H, rule)


def objective(R, mu):
    dt = mu.dtype.type
    with np.errstate(over="ignore", invalid="ignore"):
        o = dt(np.sum((np.asarray(R, mu.dtype) - mu) ** 2, dtype=mu.dtype))
    return o if np.isfinite(o) and o <= F32_MAX else dt(-np.inf)


def candidate(mu, d, g):
    return mu.copy() if g == 0 else (mu + g * d).astype(mu.dtype)


def craft(rows, slots, honest, rule, H, attack, scale, steps=STEPS):
    """(message, gamma_i*, O [steps + 1]) of the tailored attack `attack` ("tailored_uv" | "_std" | "_sgn") with range
    multiplier `scale` against a receiver with `rule` and H.  rows [n_rows, P]: the message rows; slots: the receiver's
    slot list (a row index, or -1 for a crafted slot); honest: the slot indices of the honest set."""
    rows = np.asarray(rows)
    dt = rows.dtype.type
    if attack not in ATTACKS:
        raise ValueError(f"unknown attack {attack!r}")
    if not (np.isfinite(scale) and scale >= 0):
        raise ValueError("the scale must be finite and >= 0")
    if any(slots[k] < 0 for k in honest) or -1 not in slots:
        raise ValueError("the honest slots must be real and some slot crafted")
    V = np.stack([rows[slots[k]] for k in sorted(honest)])
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    with np.errstate(over="ignore"):
        G = dt(dt(scale) * g_mm)
    if not np.isfinite(G) or abs(G) > F32_MAX:
        G = dt(0)                                        # the kernel's fp32 product overflows: Gamma = 0
    gam = [dt(dt(G * dt(i)) / dt(steps)) for i in range(steps + 1)]
    O = np.empty(steps + 1, rows.dtype)
    for i, g in enumerate(gam):
        m = candidate(mu, d, g)
        X = np.stack([m if s < 0 else rows[s] for s in slots])
        O[i] = objective(rule_output(X, rule, H), mu)
    best = int(np.argmax(O))                             # the first maximum: ties to the smaller i; all -inf: 0
    return candidate(mu, d, gam[best]), gam[best], O


def margin(O):
    """Relative margin between the best and the second-best distinct objective (inf if there is only one value)."""
    O = np.asarray(O, np.float64)
    top = np.max(O)
    rest = O[O < top]
    if not np.isfinite(top) or rest.size == 0:
        return np.inf
    return (top - np.max(rest)) / max(abs(top), 1e-300)


def make_hook(labels, in_nodes, attacks, rules, H, seed=0, round_=0, gammas=None, objectives=None):
    """attack_oracle.make_hook for attacks of every kind: attacks[b] = (name, param), with a name of rcmarl_attack,
    adaptive_attack_oracle.ATTACKS or ATTACKS.  rules[j] and H[j] are receiver j's rule and H.  gammas (a dict,
    optional) receives {(b, j): [critic gamma, TR gamma]} of the last epoch hooked, objectives {(b, j): [O critic,
    O TR]}.  Each tailored message models every Byzantine in-neighbour of j as sending it."""
    pairs = AT.byzantine_pairs(labels, in_nodes)
    # the older attacks through adaptive_attack_oracle; the tailored pairs' entries are overwritten below
    inner = AA.make_hook(labels, in_nodes, {b: (("alie", 0.0) if a[0] in ATTACKS else a) for b, a in attacks.items()},
                         seed=seed, round_=round_, gammas=gammas)
    Hs = [H] * len(labels) if np.isscalar(H) else list(H)

    def hook(epoch, critic_msgs, TR_msgs):
        dt = critic_msgs[0][0].dtype
        per_c, per_t = inner(epoch, critic_msgs, TR_msgs)
        for b, j, _ in pairs:
            name, param = attacks[b]
            if name not in ATTACKS:
                continue
            slots = [-1 if labels[i] == "Byzantine" else i for i in in_nodes[j]]
            honest = [k for k, i in enumerate(in_nodes[j]) if labels[i] == "Cooperative"]
            gs, os_ = [], []
            for msgs, per in ((critic_msgs, per_c), (TR_msgs, per_t)):
                rows = np.stack([AT.pack(msgs[i], dt) for i in range(len(labels))])
                flat, g, O = craft(rows, slots, honest, rules[j], Hs[j], name, param)
                gs.append(float(g))
                os_.append(O)
                m = AT.unpack(flat, msgs[b])
                per[j] = [m if i == b else x for i, x in zip(in_nodes[j], per[j])]
            if gammas is not None:
                gammas[(b, j)] = gs
            if objectives is not None:
                objectives[(b, j)] = os_
        return per_c, per_t
    return hook
