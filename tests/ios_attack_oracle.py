"""The IOS-aware Byzantine messages of include/rcmarl.h (rcmarl_ios_pipeline_attack, rcmarl_ios_history_attack) in
NumPy, in the dtype of the messages: the searches of pipeline_attack_oracle and history_attack_oracle, with the
receiver's clipping step (arc_oracle.clip) where `arc` is set, and the receiver's rule computed by ios_oracle (fp64
centres and distances, equal distances removing the higher index first, the mean in the messages' dtype).
craft_pipeline / craft_history return the message, gamma_i*, the objective vector, the modelled aggregate and
ios_oracle.margin of the rule's rows at the pick: the kernel sums each distance in another order, so a removal whose
margin is near 0 may go either way.  Against a receiver on mda / smea or any other rule they are subset_attack_oracle's.

make_hook gives a messages hook for attack_oracle.update_round that crafts these next to every older attack (an ios_*
pair against a receiver that is not on ios is subset_attack_oracle's, as in the Trainer); chain_hook composes it with
the momentum, ARC and mixing hooks in the trainer's order, as subset_attack_oracle.chain_hook does."""
import numpy as np

import arc_attack_oracle as AAO
import arc_oracle as AO
import attack_oracle as AT
import bucket_oracle as BO
import ios_oracle as IO
import momentum_oracle as MO
import nnm_oracle as NO
import pipeline_attack_oracle as PA
import subset_attack_oracle as SAO

STEPS = SAO.STEPS
ATTACKS = tuple(f"ios_{d}" for d in ("uv", "std", "sgn"))


def as_subset(attack):
    """The subset attack in the same direction: what an ios_* attacker sends a receiver that is not on ios."""
    return "subset_" + attack.split("_")[1]


def rule_output(X, rule, H):
    """R_j(X): ios_oracle.aggregate for "ios", subset_attack_oracle.rule_output for any other rule."""
    return IO.aggregate(X, H)[0] if rule == "ios" else SAO.rule_output(X, rule, H)


def _check(attack, scale, slots, honest, arc):
    if attack not in ATTACKS:
        raise ValueError(f"unknown attack {attack!r}")
    if not (np.isfinite(scale) and scale >= 0):
        raise ValueError("the scale must be finite and >= 0")
    if any(slots[k] < 0 for k in honest) or -1 not in slots or (arc and slots[0] < 0):
        raise ValueError("the honest slots (and slot 0 under ARC) must be real, and some slot crafted")


def craft_pipeline(rows, slots, honest, rule, H, attack, scale, mixing=None, n_perms=1, arc=False, seed=0, attacker=0,
                   receiver=0, net=0, round_=0, epoch=0, follow=None, gap=1e-4):
    """(message, gamma_i*, Obar [STEPS + 1], R_0(gamma_i*), margin) of the pipeline form against a receiver that runs
    [ARC] -> `mixing` -> `rule` at H; the other arguments are pipeline_attack_oracle.craft's."""
    if rule != "ios":
        _check(attack, scale, slots, honest, arc)
        return SAO.craft_pipeline(rows, slots, honest, rule, H, as_subset(attack), scale, mixing, n_perms, arc, seed,
                                  attacker, receiver, net, round_, epoch, follow, gap)
    rows = np.asarray(rows)
    dt = rows.dtype.type
    _check(attack, scale, slots, honest, arc)
    bucket = isinstance(mixing, tuple)
    nq = n_perms if bucket else 1
    bks = [PA.buckets(len(slots), mixing[1], seed, q, attacker, receiver, net, round_, epoch) if bucket else None
           for q in range(nq)]
    mu, d, gam = AAO._candidates(np.stack([rows[slots[k]] for k in sorted(honest)]), attack, scale, dt)

    def mixed(g, q):
        m = SAO.TA.candidate(mu, d, g)
        return PA.mix(SAO._clip(np.stack([m if s < 0 else rows[s] for s in slots]), H, arc), mixing, H, bks[q])
    Ob = np.empty(STEPS + 1, rows.dtype)
    for i, g in enumerate(gam):
        with np.errstate(over="ignore", invalid="ignore"):
            acc = dt(0)
            for q in range(nq):                          # q order, from 0
                acc = dt(acc + SAO.TA.objective(rule_output(mixed(g, q), rule, H), mu))
            ob = dt(acc / dt(nq))
        Ob[i] = ob if np.isfinite(ob) and ob <= SAO.TA.F32_MAX else dt(-np.inf)
    best = AAO._pick(Ob, gam, follow, gap)
    Z = mixed(gam[best], 0)
    return (SAO.TA.candidate(mu, d, gam[best]), gam[best], Ob, np.asarray(rule_output(Z, rule, H), rows.dtype),
            IO.margin(Z, H))


def craft_history(rows, slots, honest, rule, H, attack, scale, c, M, beta, first, own, arc=False, follow=None,
                  gap=1e-4):
    """(message, gamma_i*, O [STEPS + 1], R(gamma_i*), margin) of the history form against a receiver that runs
    momentum -> [ARC] -> `rule` at H; the other arguments are history_attack_oracle.craft's."""
    if rule != "ios":
        _check(attack, scale, slots, honest, arc)
        return SAO.craft_history(rows, slots, honest, rule, H, as_subset(attack), scale, c, M, beta, first, own, arc,
                                 follow, gap)
    rows = np.asarray(rows)
    dt = rows.dtype.type
    _check(attack, scale, slots, honest, arc)
    crafted = [k for k, s in enumerate(slots) if s < 0]
    own = sorted(set(own))
    if not own or any(k not in crafted for k in own):
        raise ValueError("the own slots must be crafted, and at least one")
    k0 = own[0]
    c = np.asarray(c, rows.dtype)
    Mk = (lambda k: None) if first else (lambda k: np.asarray(M[k], rows.dtype))
    Y = np.stack([SAO.HO.step_row(rows[s], c, Mk(k), beta, first) if s >= 0 else np.zeros_like(c)
                  for k, s in enumerate(slots)])
    mu, d, gam = AAO._candidates(Y[sorted(honest)], attack, scale, dt)

    def model(g):
        t = SAO.TA.candidate(mu, d, g)
        msgs = {k: SAO.HO.invert(t, c, Mk(k0 if k in own else k), beta, first) for k in crafted}
        X = Y.copy()
        for k in crafted:
            X[k] = SAO.HO.step_row(msgs[k], c, Mk(k), beta, first)
        ok = all(np.isfinite(m).all() for m in msgs.values())
        return msgs[k0], SAO._clip(X, H, arc), ok
    O = np.empty(STEPS + 1, rows.dtype)
    for i, g in enumerate(gam):
        _, Z, ok = model(g)
        O[i] = SAO.TA.objective(rule_output(Z, rule, H), mu) if ok else dt(-np.inf)
    best = AAO._pick(O, gam, follow, gap)
    m, Z, _ = model(gam[best])
    return m, gam[best], O, np.asarray(rule_output(Z, rule, H), rows.dtype), IO.margin(Z, H)


def make_hook(agents, labels, in_nodes, attacks, rules, H, momentum, mixing, clipping, seed=0, round_=0,
              n_perms=PA.PERMS, gammas=None, follow=None, gap=1e-4):
    """subset_attack_oracle.make_hook for attacks of every kind: attacks[b] = (name, param) with a name of
    subset_attack_oracle.make_hook or ATTACKS.  An IOS pair (b, j) whose receiver is on ios crafts as the Trainer does:
    the history form through j's momentum (c = agents[j]'s nets, M and first from the bound MomentumHook `hook.state`)
    and clipping if j has momentum, else the pipeline form through j's clipping and mixing; against any other receiver
    it is the subset attack in the same direction (so the ARC attack against a receiver on neither mda nor smea).
    gammas / follow / gap as in arc_attack_oracle."""
    pairs = AT.byzantine_pairs(labels, in_nodes)
    mix = [None] * len(labels) if mixing is None else list(mixing)
    clip = [None] * len(labels) if clipping is None else list(clipping)
    as_sub = {b: ((as_subset(a[0]), a[1]) if a[0] in ATTACKS else a) for b, a in attacks.items()}
    # the inner hook crafts every pair; those of the IOS pairs against ios (modelled there as clip) are replaced below
    inner = SAO.make_hook(agents, labels, in_nodes, as_sub, ["clip" if r == "ios" else r for r in rules], H, momentum,
                          mix, clip, seed=seed, round_=round_, n_perms=n_perms, gammas=gammas, follow=follow, gap=gap)
    Hs = [H] * len(labels) if np.isscalar(H) else list(H)

    def hook(epoch, critic_msgs, TR_msgs):
        inner.state = hook.state
        dt = critic_msgs[0][0].dtype
        per_c, per_t = inner(epoch, critic_msgs, TR_msgs)
        for b, j, _ in pairs:
            name, param = attacks[b]
            if name not in ATTACKS or rules[j] != "ios":
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
                    flat, g = craft_history(rows, slots, honest, "ios", Hs[j], name, param, c, M, momentum[j],
                                            M is None, own, arc=clip[j] is not None, follow=fol, gap=gap)[:2]
                else:
                    flat, g = craft_pipeline(rows, slots, honest, "ios", Hs[j], name, param, mixing=mix[j],
                                             n_perms=n_perms, arc=clip[j] is not None, seed=seed, attacker=b,
                                             receiver=j, net=net, round_=round_, epoch=epoch, follow=fol, gap=gap)[:2]
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
    """make_hook inside the receivers' chain in the trainer's order (subset_attack_oracle.chain_hook's): the attack
    hook, then MomentumHook (bound to it), ArcHook, and the nnm or bucketing hook of the receivers that mix."""
    Hs = [H] * len(labels) if np.isscalar(H) else list(H)
    mix = [None] * len(labels) if mixing is None else list(mixing)
    clip = [None] * len(labels) if clipping is None else list(clipping)
    inner = make_hook(agents, labels, in_nodes, attacks, rules, Hs, momentum, mix, clip, seed=seed, round_=round_,
                      **kw)
    mh = MO.MomentumHook(agents, labels, in_nodes, momentum, inner=inner)
    inner.state = mh
    out = AO.ArcHook(labels, in_nodes, clip, Hs, inner=mh)
    if any(m == "nnm" for m in mix):
        out = NO.mixing_hook(labels, in_nodes, [m if m == "nnm" else None for m in mix], Hs, inner=out,
                             kernel_M=kernel_M)
    if any(isinstance(m, tuple) for m in mix):
        out = BO.bucketing_hook(labels, in_nodes, [m if isinstance(m, tuple) else None for m in mix], seed, round_,
                                inner=out)
    return out


update_round = AT.update_round
