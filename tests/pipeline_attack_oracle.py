"""The pipeline-aware Byzantine messages of include/rcmarl.h (rcmarl_pipeline_attack) in NumPy, in the dtype of the
messages (fp32 or fp64), built on tailored_attack_oracle (mu, d, the candidates and the objective), nnm_oracle and
bucket_oracle (the mixing step) and dnc_oracle (the spectral rule): craft() returns the message, gamma_i*, the mean
objective vector Obar and the modelled aggregate R_0(gamma_i*); and a messages hook for attack_oracle.update_round that
crafts these next to the attacks of tailored_attack_oracle.make_hook, and composes with nnm_oracle.mixing_hook and
bucket_oracle.bucketing_hook around it.

As in the kernel, an objective that is not finite or exceeds the fp32 range counts as -inf in either dtype."""
import numpy as np

import adaptive_attack_oracle as AA
import attack_oracle as AT
import bucket_oracle as BO
import dnc_oracle as DO
import nnm_oracle as NO
import tailored_attack_oracle as TA

STEPS = TA.STEPS
ATTACKS = tuple(f"pipeline_{d}" for d in AA.DEVS)
RULES = TA.RULES + ("dnc",)
STREAM = 0x10000000                                    # bit 28 of counter word 1
MAX_PERMS = 16                                         # RCMARL_PIPELINE_MAX_PERMS
PERMS = 4                                              # the trainer's samples (L.PIPELINE_PERMS)


def counter(q, t, attacker, receiver, net, round_, epoch):
    """The Philox counter of draw t of the attacker's shuffle sample q."""
    return ((q << 2) | (t >> 2), attacker | receiver << 8 | net << 16 | STREAM, round_ & 0xFFFFFFFF, epoch & 0xFFFFFFFF)


def draws(count, seed, q, attacker, receiver, net, round_, epoch):
    """The first `count` 32-bit draws of sample q: draw t is word t & 3 of Philox4x32-10 at counter(q, t, ...) under
    key (seed low word, seed high word)."""
    if not (0 <= q < MAX_PERMS and 0 <= attacker <= 255 and 0 <= receiver <= 255 and net in (0, 1)):
        raise ValueError("the sample and the counter words are out of range")
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if count <= 0:
        return []
    ctr = [np.array([counter(q, 4 * c, attacker, receiver, net, round_, epoch)[w] for c in range((count + 3) // 4)],
                    np.uint64) for w in range(4)]
    words = AT.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    return [int(words[t & 3][t >> 2]) for t in range(count)]


def buckets(n_in, s, seed, q, attacker, receiver, net, round_, epoch):
    """The buckets of sample q, each in increasing slot order: bucket_oracle's Fisher-Yates and bucketing on draws()."""
    BO.n_out(n_in, s)
    m = n_in - 1
    pi = list(range(1, m + 1))
    u = draws(m - 1, seed, q, attacker, receiver, net, round_, epoch)
    for t, i in enumerate(range(m - 1, 0, -1)):
        j = (u[t] * (i + 1)) >> 32
        pi[i], pi[j] = pi[j], pi[i]
    return [sorted(pi[b:b + s]) for b in range(0, m, s)]


def mix(X, mixing, H, bks=None):
    """The rows the receiver's rule reads: X itself (mixing None), nnm_oracle's mixed rows ("nnm") or bucket_oracle's
    rows of the buckets bks (("bucket", s))."""
    if mixing is None:
        return X
    if mixing == "nnm":
        return NO.mix(X, H)[0]
    return BO.mix(X, bks)[0]


def rule_output(X, rule, H):
    """R_j(X) of the receiver's rule over the rows X, DnC included."""
    return DO.aggregate(X, H)[0] if rule == "dnc" else TA.rule_output(X, rule, H)


def n_rows(n_in, mixing):
    return BO.n_out(n_in, mixing[1]) if isinstance(mixing, tuple) else n_in


def craft(rows, slots, honest, rule, H, attack, scale, mixing=None, n_perms=1, seed=0, attacker=0, receiver=0, net=0,
          round_=0, epoch=0, follow=None, gap=1e-4):
    """(message, gamma_i*, Obar [STEPS + 1], R_0(gamma_i*)) of the pipeline attack `attack` ("pipeline_uv" | "_std" |
    "_sgn") with range multiplier `scale` against a receiver with `mixing` (None, "nnm" or ("bucket", s)), `rule` and H.
    rows [n_rows, P]: the message rows; slots: the receiver's slot list (a row index, or -1 for a crafted slot); honest:
    the slot indices of the honest set.  Under bucketing Obar averages the n_perms samples drawn from (seed, attacker,
    receiver, net, round_, epoch); otherwise there is one sample.  follow (the kernel's gamma_i*, optional): where the
    relative margin of Obar is at most `gap`, the pick is the candidate nearest to it if its Obar lies within `gap`
    relative of the maximum -- a near tie that fp32 may break either way."""
    rows = np.asarray(rows)
    dt = rows.dtype.type
    if attack not in ATTACKS:
        raise ValueError(f"unknown attack {attack!r}")
    if not (np.isfinite(scale) and scale >= 0):
        raise ValueError("the scale must be finite and >= 0")
    if any(slots[k] < 0 for k in honest) or -1 not in slots:
        raise ValueError("the honest slots must be real and some slot crafted")
    bucket = isinstance(mixing, tuple)
    if bucket and not 1 <= n_perms <= MAX_PERMS:
        raise ValueError(f"n_perms must lie in 1 .. {MAX_PERMS}")
    nq = n_perms if bucket else 1
    bks = [buckets(len(slots), mixing[1], seed, q, attacker, receiver, net, round_, epoch) if bucket else None
           for q in range(nq)]
    V = np.stack([rows[slots[k]] for k in sorted(honest)])
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    with np.errstate(over="ignore"):
        G = dt(dt(scale) * g_mm)
    if not np.isfinite(G) or abs(G) > TA.F32_MAX:
        G = dt(0)                                        # the kernel's fp32 product overflows: Gamma = 0
    gam = [dt(dt(G * dt(i)) / dt(STEPS)) for i in range(STEPS + 1)]

    def model(g, q):
        m = TA.candidate(mu, d, g)
        X = np.stack([m if s < 0 else rows[s] for s in slots])
        return rule_output(mix(X, mixing, H, bks[q]), rule, H)
    Ob = np.empty(STEPS + 1, rows.dtype)
    for i, g in enumerate(gam):
        O = [TA.objective(model(g, q), mu) for q in range(nq)]
        with np.errstate(over="ignore", invalid="ignore"):
            acc = dt(0)
            for o in O:                                  # q order, from 0
                acc = dt(acc + o)
            ob = dt(acc / dt(nq))
        Ob[i] = ob if np.isfinite(ob) and ob <= TA.F32_MAX else dt(-np.inf)
    best = int(np.argmax(Ob))                            # the first maximum: ties to the smaller i; all -inf: 0
    if follow is not None and margin(Ob) <= gap:
        k = int(np.argmin([abs(float(g) - float(follow)) for g in gam]))
        if Ob[k] >= Ob[best] - gap * abs(Ob[best]):
            best = k
    return TA.candidate(mu, d, gam[best]), gam[best], Ob, np.asarray(model(gam[best], 0), rows.dtype)


margin = TA.margin


def make_hook(labels, in_nodes, attacks, rules, H, mixing, seed=0, round_=0, n_perms=PERMS, gammas=None,
              objectives=None, follow=None):
    """attack_oracle.make_hook for attacks of every kind: attacks[b] = (name, param), with a name of rcmarl_attack,
    adaptive_attack_oracle.ATTACKS, tailored_attack_oracle.ATTACKS or ATTACKS.  rules[j], H[j] and mixing[j] are
    receiver j's rule, H and mixing entry; the pipeline pairs draw their samples as the Trainer does (attacker b,
    receiver j, net 0 critic / 1 TR, seed, round_, the epoch).  gammas / objectives (dicts, optional) receive
    {(b, j): [critic, TR]} of the last epoch hooked.  follow[epoch][(b, j)] ([2], e.g. Trainer.attack_gammas() of a
    run whose last epoch is `epoch`), when given, supplies the kernel's gamma for craft's near ties.  Wrap the result
    in the receivers' mixing hooks."""
    pairs = AT.byzantine_pairs(labels, in_nodes)
    inner = TA.make_hook(labels, in_nodes, {b: (("alie", 0.0) if a[0] in ATTACKS else a) for b, a in attacks.items()},
                         rules, H, seed=seed, round_=round_, gammas=gammas, objectives=objectives)
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
            for net, (msgs, per) in enumerate(((critic_msgs, per_c), (TR_msgs, per_t))):
                rows = np.stack([AT.pack(msgs[i], dt) for i in range(len(labels))])
                kg = (follow or {}).get(epoch, {}).get((b, j))
                flat, g, O, _ = craft(rows, slots, honest, rules[j], Hs[j], name, param, mixing=mixing[j],
                                      n_perms=n_perms, seed=seed, attacker=b, receiver=j, net=net, round_=round_,
                                      epoch=epoch, follow=None if kg is None else kg[net])
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


update_round = AT.update_round
