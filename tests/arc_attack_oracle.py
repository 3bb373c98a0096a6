"""The ARC-aware Byzantine messages of include/rcmarl.h (rcmarl_pipeline_arc_attack, rcmarl_history_arc_attack) in
NumPy, in the dtype of the messages: the searches of pipeline_attack_oracle and history_attack_oracle with the
receiver's clipping step (arc_oracle.clip: fp64 factors, the rows in the messages' dtype) inserted before the mixing
step (pipeline form) or between the momentum rows and the rule (history form).  craft_pipeline / craft_history return
the message, gamma_i*, the objective vector, the modelled aggregate and the crafted slots' clipping factors at the pick.

make_hook gives a messages hook for attack_oracle.update_round that crafts these next to every older attack;
chain_hook composes it with momentum_oracle.MomentumHook, arc_oracle.ArcHook and the mixing hooks in the trainer's
order (attack -> momentum -> ARC -> nnm | bucketing).  An arc_* pair whose receiver does not clip is the history attack
in the same direction, as in the Trainer."""
import numpy as np

import adaptive_attack_oracle as AA
import arc_oracle as AO
import attack_oracle as AT
import bucket_oracle as BO
import history_attack_oracle as HO
import momentum_oracle as MO
import nnm_oracle as NO
import pipeline_attack_oracle as PA
import tailored_attack_oracle as TA

STEPS = TA.STEPS
ATTACKS = tuple(f"arc_{d}" for d in AA.DEVS)


def _check(attack, scale, slots, honest):
    if attack not in ATTACKS:
        raise ValueError(f"unknown attack {attack!r}")
    if not (np.isfinite(scale) and scale >= 0):
        raise ValueError("the scale must be finite and >= 0")
    if any(slots[k] < 0 for k in honest) or -1 not in slots or slots[0] < 0:
        raise ValueError("the honest slots and slot 0 must be real, and some slot crafted")


def _candidates(V, attack, scale, dt):
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    with np.errstate(over="ignore"):
        G = dt(dt(scale) * g_mm)
    if not np.isfinite(G) or abs(G) > TA.F32_MAX:
        G = dt(0)                                        # the kernel's fp32 product overflows: Gamma = 0
    return mu, d, [dt(dt(G * dt(i)) / dt(STEPS)) for i in range(STEPS + 1)]


def _pick(O, gam, follow, gap):
    best = int(np.argmax(O))                             # the first maximum: ties to the smaller i; all -inf: 0
    if follow is not None and TA.margin(O) <= gap:
        k = int(np.argmin([abs(float(g) - float(follow)) for g in gam]))
        if O[k] >= O[best] - gap * abs(O[best]):
            best = k
    return best


def craft_pipeline(rows, slots, honest, rule, H, attack, scale, mixing=None, n_perms=1, seed=0, attacker=0, receiver=0,
                   net=0, round_=0, epoch=0, follow=None, gap=1e-4):
    """(message, gamma_i*, Obar [STEPS + 1], R_0(gamma_i*), c of the crafted slots at the pick) of the pipeline form
    against a receiver that clips at H before `mixing` and `rule`; the arguments are pipeline_attack_oracle.craft's."""
    rows = np.asarray(rows)
    dt = rows.dtype.type
    _check(attack, scale, slots, honest)
    bucket = isinstance(mixing, tuple)
    nq = n_perms if bucket else 1
    bks = [PA.buckets(len(slots), mixing[1], seed, q, attacker, receiver, net, round_, epoch) if bucket else None
           for q in range(nq)]
    mu, d, gam = _candidates(np.stack([rows[slots[k]] for k in sorted(honest)]), attack, scale, dt)

    def clipped(g):
        m = TA.candidate(mu, d, g)
        return AO.clip(np.stack([m if s < 0 else rows[s] for s in slots]), H)[:2]

    def model(Y, q):
        return PA.rule_output(PA.mix(Y, mixing, H, bks[q]), rule, H)
    Ob = np.empty(STEPS + 1, rows.dtype)
    for i, g in enumerate(gam):
        Y = clipped(g)[0]
        with np.errstate(over="ignore", invalid="ignore"):
            acc = dt(0)
            for q in range(nq):                          # q order, from 0
                acc = dt(acc + TA.objective(model(Y, q), mu))
            ob = dt(acc / dt(nq))
        Ob[i] = ob if np.isfinite(ob) and ob <= TA.F32_MAX else dt(-np.inf)
    best = _pick(Ob, gam, follow, gap)
    Y, c = clipped(gam[best])
    return (TA.candidate(mu, d, gam[best]), gam[best], Ob, np.asarray(model(Y, 0), rows.dtype),
            c[[k for k, s in enumerate(slots) if s < 0]])


def craft_history(rows, slots, honest, rule, H, attack, scale, c, M, beta, first, own, follow=None, gap=1e-4):
    """(message, gamma_i*, O [STEPS + 1], R(gamma_i*), c of the crafted slots at the pick) of the history form against
    a receiver that clips at H between its momentum rows and `rule`; the arguments are history_attack_oracle.craft's."""
    rows = np.asarray(rows)
    dt = rows.dtype.type
    _check(attack, scale, slots, honest)
    crafted = [k for k, s in enumerate(slots) if s < 0]
    own = sorted(set(own))
    if not own or any(k not in crafted for k in own):
        raise ValueError("the own slots must be crafted, and at least one")
    k0 = own[0]
    c = np.asarray(c, rows.dtype)
    Mk = (lambda k: None) if first else (lambda k: np.asarray(M[k], rows.dtype))
    Y = np.stack([HO.step_row(rows[s], c, Mk(k), beta, first) if s >= 0 else np.zeros_like(c)
                  for k, s in enumerate(slots)])
    mu, d, gam = _candidates(Y[sorted(honest)], attack, scale, dt)

    def model(g):
        t = TA.candidate(mu, d, g)
        msgs = {k: HO.invert(t, c, Mk(k0 if k in own else k), beta, first) for k in crafted}
        X = Y.copy()
        for k in crafted:
            X[k] = HO.step_row(msgs[k], c, Mk(k), beta, first)
        ok = all(np.isfinite(m).all() for m in msgs.values())
        Z, f = AO.clip(X, H)[:2]
        return msgs[k0], PA.rule_output(Z, rule, H), ok, f
    O = np.empty(STEPS + 1, rows.dtype)
    for i, g in enumerate(gam):
        _, R, ok, _ = model(g)
        O[i] = TA.objective(R, mu) if ok else dt(-np.inf)
    best = _pick(O, gam, follow, gap)
    m, R, _, f = model(gam[best])
    return m, gam[best], O, np.asarray(R, rows.dtype), f[crafted]


def make_hook(agents, labels, in_nodes, attacks, rules, H, momentum, mixing, clipping, seed=0, round_=0,
              n_perms=PA.PERMS, gammas=None, follow=None, gap=1e-4):
    """attack_oracle.make_hook for attacks of every kind: attacks[b] = (name, param) with a name of
    history_attack_oracle.make_hook or ATTACKS.  An ARC pair (b, j) crafts as the Trainer does: through j's momentum
    (c = agents[j]'s nets, M and first from the bound MomentumHook `hook.state`) and clipping if j has both, through
    j's clipping and mixing if j clips without momentum, and as the history attack if j does not clip.  gammas /
    follow as in history_attack_oracle.make_hook; gap: the near-tie bound of craft_pipeline / craft_history for the ARC
    pairs."""
    pairs = AT.byzantine_pairs(labels, in_nodes)
    mix = [None] * len(labels) if mixing is None else list(mixing)
    as_hist = {b: (("history_" + a[0].split("_")[1], a[1]) if a[0] in ATTACKS else a) for b, a in attacks.items()}
    inner = HO.make_hook(agents, labels, in_nodes, as_hist, rules, H, momentum, mixing=mix, seed=seed, round_=round_,
                         n_perms=n_perms, gammas=gammas, follow=follow)
    Hs = [H] * len(labels) if np.isscalar(H) else list(H)

    def hook(epoch, critic_msgs, TR_msgs):
        inner.state = hook.state
        dt = critic_msgs[0][0].dtype
        per_c, per_t = inner(epoch, critic_msgs, TR_msgs)
        for b, j, _ in pairs:
            name, param = attacks[b]
            if name not in ATTACKS or clipping[j] is None:
                continue
            slots = [-1 if labels[i] == "Byzantine" else i for i in in_nodes[j]]
            honest = [k for k, i in enumerate(in_nodes[j]) if labels[i] == "Cooperative"]
            gs = []
            for net, (msgs, per) in enumerate(((critic_msgs, per_c), (TR_msgs, per_t))):
                rows = np.stack([AT.pack(msgs[i], dt) for i in range(len(labels))])
                kg = (follow or {}).get(epoch, {}).get((b, j))
                fol = None if kg is None else kg[net]
                if momentum[j] is not None:
                    own = [k for k, i in enumerate(in_nodes[j]) if i == b]
                    c = AT.pack(agents[j].get_parameters()[1 + net], dt)
                    M = hook.state.M.get((j, net))
                    flat, g = craft_history(rows, slots, honest, rules[j], Hs[j], name, param, c, M, momentum[j],
                                            M is None, own, follow=fol, gap=gap)[:2]
                else:
                    flat, g = craft_pipeline(rows, slots, honest, rules[j], Hs[j], name, param, mixing=mix[j],
                                             n_perms=n_perms, seed=seed, attacker=b, receiver=j, net=net,
                                             round_=round_, epoch=epoch, follow=fol, gap=gap)[:2]
                gs.append(float(g))
                m = AT.unpack(flat, msgs[b])
                per[j] = [m if i == b else x for i, x in zip(in_nodes[j], per[j])]
            if gammas is not None:
                gammas[(b, j)] = gs
        return per_c, per_t
    hook.state = None
    return hook


def chain_hook(agents, labels, in_nodes, attacks, rules, H, momentum, mixing, clipping, seed=0, round_=0,
               kernel_M=None, **kw):
    """make_hook inside the receivers' chain in the trainer's order: the attack hook, then MomentumHook (bound to it:
    the attack reads each receiver's M before that epoch's step), ArcHook, and the nnm or bucketing hook of the
    receivers that mix (kernel_M as for nnm_oracle.mixing_hook)."""
    Hs = [H] * len(labels) if np.isscalar(H) else list(H)
    mix = [None] * len(labels) if mixing is None else list(mixing)
    inner = make_hook(agents, labels, in_nodes, attacks, rules, Hs, momentum, mix, clipping, seed=seed, round_=round_,
                      **kw)
    mh = MO.MomentumHook(agents, labels, in_nodes, momentum, inner=inner)
    inner.state = mh
    out = AO.ArcHook(labels, in_nodes, clipping, Hs, inner=mh)
    if any(m == "nnm" for m in mix):
        out = NO.mixing_hook(labels, in_nodes, [m if m == "nnm" else None for m in mix], Hs, inner=out,
                             kernel_M=kernel_M)
    if any(isinstance(m, tuple) for m in mix):
        out = BO.bucketing_hook(labels, in_nodes, [m if isinstance(m, tuple) else None for m in mix], seed, round_,
                                inner=out)
    return out


update_round = AT.update_round
