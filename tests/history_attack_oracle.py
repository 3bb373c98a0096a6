"""The momentum-aware Byzantine messages of include/rcmarl.h (rcmarl_history_attack) in NumPy, in the dtype of the
messages (fp32 or fp64).  The receiver's momentum step is momentum_oracle.step and the inversion is restated here; in
fp32 both round every operation on its own, as the kernel does, so they match it bit for bit.  The search (mu, d,
gamma_mm, the candidates, the rules and the objective) is that of pipeline_attack_oracle / tailored_attack_oracle
without mixing, run on the momentum rows: craft() returns the message, gamma_i*, the objective vector O, the modelled
aggregate R(gamma_i*) and the modelled rows.

make_hook gives a messages hook for attack_oracle.update_round that crafts these next to every older attack, and
momentum_hook wraps it in momentum_oracle.MomentumHook: the attack reads each receiver's M before that epoch's step.

As in the kernel, an objective that is not finite or exceeds the fp32 range counts as -inf in either dtype, and so
does a candidate whose crafted messages are not all finite."""
import numpy as np

import adaptive_attack_oracle as AA
import attack_oracle as AT
import momentum_oracle as MO
import pipeline_attack_oracle as PA
import tailored_attack_oracle as TA

STEPS = TA.STEPS
ATTACKS = tuple(f"history_{d}" for d in AA.DEVS)
RULES = PA.RULES
MAX_FLOATS = 22 * 1421                                 # RCMARL_HISTORY_MAX_FLOATS


def invert(t, c, M, beta, first):
    """The message that puts a slot's momentum row at t [P] (include/rcmarl.h, Inversion), in t's dtype: t where first
    or M is +-inf, else c + ((t - c) - beta M) / (1 - beta), each operation rounded on its own.  M is not read when
    first."""
    t = np.asarray(t)
    if first:
        return t.copy()
    dt = t.dtype.type
    c, M, b = np.asarray(c, t.dtype), np.asarray(M, t.dtype), dt(beta)
    with np.errstate(over="ignore", invalid="ignore"):
        m = c + ((t - c) - b * M) / (dt(1) - b)
    return np.where(np.isinf(M), t, m).astype(t.dtype)


def step_row(x, c, Mk, beta, first):
    """One slot's momentum row step_k(x) [P]: momentum_oracle.step on that slot alone."""
    return MO.step(np.asarray(x)[None], c, None if first else np.asarray(Mk)[None], beta, first)[0][0]


def craft(rows, slots, honest, rule, H, attack, scale, c, M, beta, first, own, follow=None, gap=1e-4):
    """(message, gamma_i*, O [STEPS + 1], R(gamma_i*), the modelled rows [n_in, P]) of the history attack `attack`
    ("history_uv" | "_std" | "_sgn") with range multiplier `scale` against a receiver with `rule` and H.  rows [n, P]:
    the message rows; slots: the receiver's slot list (a row index, or -1 for a crafted slot); honest: the slot indices
    of the honest set; c [P]: the receiver's reference; M [>= n_in, P]: its state, row k slot k's (not read when
    first); beta; first; own: the crafted slots that receive the message.  follow (the kernel's gamma_i*, optional):
    at a near tie, as pipeline_attack_oracle.craft."""
    rows = np.asarray(rows)
    dt = rows.dtype.type
    if attack not in ATTACKS:
        raise ValueError(f"unknown attack {attack!r}")
    if not (np.isfinite(scale) and scale >= 0):
        raise ValueError("the scale must be finite and >= 0")
    if any(slots[k] < 0 for k in honest) or -1 not in slots:
        raise ValueError("the honest slots must be real and some slot crafted")
    crafted = [k for k, s in enumerate(slots) if s < 0]
    own = sorted(set(own))
    if not own or any(k not in crafted for k in own):
        raise ValueError("the own slots must be crafted, and at least one")
    k0 = own[0]
    c = np.asarray(c, rows.dtype)
    Mk = (lambda k: None) if first else (lambda k: np.asarray(M[k], rows.dtype))
    Y = np.stack([step_row(rows[s], c, Mk(k), beta, first) if s >= 0 else np.zeros_like(c)
                  for k, s in enumerate(slots)])
    V = Y[sorted(honest)]
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    with np.errstate(over="ignore"):
        G = dt(dt(scale) * g_mm)
    if not np.isfinite(G) or abs(G) > TA.F32_MAX:
        G = dt(0)                                        # the kernel's fp32 product overflows: Gamma = 0
    gam = [dt(dt(G * dt(i)) / dt(STEPS)) for i in range(STEPS + 1)]

    def model(g):
        t = TA.candidate(mu, d, g)
        msgs = {k: invert(t, c, Mk(k0 if k in own else k), beta, first) for k in crafted}
        X = Y.copy()
        for k in crafted:
            X[k] = step_row(msgs[k], c, Mk(k), beta, first)
        ok = all(np.isfinite(m).all() for m in msgs.values())
        return msgs[k0], PA.rule_output(X, rule, H), X, ok
    O = np.empty(STEPS + 1, rows.dtype)
    for i, g in enumerate(gam):
        _, R, _, ok = model(g)
        O[i] = TA.objective(R, mu) if ok else dt(-np.inf)
    best = int(np.argmax(O))                             # the first maximum: ties to the smaller i; all -inf: 0
    if follow is not None and TA.margin(O) <= gap:
        k = int(np.argmin([abs(float(g) - float(follow)) for g in gam]))
        if O[k] >= O[best] - gap * abs(O[best]):
            best = k
    m, R, X, _ = model(gam[best])
    return m, gam[best], O, np.asarray(R, rows.dtype), X


def make_hook(agents, labels, in_nodes, attacks, rules, H, momentum, mixing=None, seed=0, round_=0,
              n_perms=PA.PERMS, gammas=None, follow=None):
    """attack_oracle.make_hook for attacks of every kind: attacks[b] = (name, param) with a name of
    pipeline_attack_oracle.make_hook or ATTACKS.  A history pair (b, j) whose receiver has momentum[j] not None crafts
    through j's momentum as the Trainer does (c = agents[j]'s nets, M and first from the bound MomentumHook `hook.state`,
    own = every slot of b in in_nodes[j]); one whose receiver has no momentum is the pipeline attack in the same
    direction.  gammas (a dict, optional) receives {(b, j): [critic, TR]} of the last epoch hooked; follow[epoch][(b, j)]
    supplies the kernel's gamma for near ties.  Use momentum_hook to bind the state."""
    pairs = AT.byzantine_pairs(labels, in_nodes)
    mix = [None] * len(labels) if mixing is None else list(mixing)
    as_pipe = {b: (("pipeline_" + a[0].split("_")[1], a[1]) if a[0] in ATTACKS else a) for b, a in attacks.items()}
    inner = PA.make_hook(labels, in_nodes, as_pipe, rules, H, mix, seed=seed, round_=round_, n_perms=n_perms,
                         gammas=gammas, follow=follow)
    Hs = [H] * len(labels) if np.isscalar(H) else list(H)

    def hook(epoch, critic_msgs, TR_msgs):
        dt = critic_msgs[0][0].dtype
        per_c, per_t = inner(epoch, critic_msgs, TR_msgs)
        for b, j, _ in pairs:
            name, param = attacks[b]
            if name not in ATTACKS or momentum[j] is None:
                continue
            slots = [-1 if labels[i] == "Byzantine" else i for i in in_nodes[j]]
            honest = [k for k, i in enumerate(in_nodes[j]) if labels[i] == "Cooperative"]
            own = [k for k, i in enumerate(in_nodes[j]) if i == b]
            gs = []
            for net, (msgs, per) in enumerate(((critic_msgs, per_c), (TR_msgs, per_t))):
                rows = np.stack([AT.pack(msgs[i], dt) for i in range(len(labels))])
                c = AT.pack(agents[j].get_parameters()[1 + net], dt)
                M = hook.state.M.get((j, net))
                kg = (follow or {}).get(epoch, {}).get((b, j))
                flat, g, _, _, _ = craft(rows, slots, honest, rules[j], Hs[j], name, param, c, M, momentum[j],
                                         M is None, own, follow=None if kg is None else kg[net])
                gs.append(float(g))
                m = AT.unpack(flat, msgs[b])
                per[j] = [m if i == b else x for i, x in zip(in_nodes[j], per[j])]
            if gammas is not None:
                gammas[(b, j)] = gs
        return per_c, per_t
    hook.state = None
    return hook


def momentum_hook(agents, labels, in_nodes, attacks, rules, H, momentum, mixing=None, log=None, **kw):
    """momentum_oracle.MomentumHook around make_hook's attack hook, bound to it: within one epoch the attack reads each
    receiver's M before the momentum step of that epoch."""
    inner = make_hook(agents, labels, in_nodes, attacks, rules, H, momentum, mixing=mixing, **kw)
    mh = MO.MomentumHook(agents, labels, in_nodes, momentum, inner=inner, log=log)
    inner.state = mh
    return mh


update_round = AT.update_round
