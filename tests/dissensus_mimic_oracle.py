"""The dissensus and mimic Byzantine messages of include/rcmarl.h (rcmarl_dissensus_attack, rcmarl_mimic_attack) in
NumPy, in the dtype of the messages (fp32 or fp64); and a messages hook for attack_oracle.update_round that crafts them
next to the attacks of tailored_attack_oracle.make_hook, so that it composes with the agents of agg_oracle,
vector_oracle and dnc_oracle and with nnm_oracle.mixing_hook.  The mimic hook is an object: it carries each
(attacker, receiver, net)'s direction z and each pair's power-step count across epochs and rounds.

As in the kernel, a sum over the parameters that is not finite or exceeds the fp32 range counts as +inf in either dtype
(a mimic score t_k as -inf)."""
import numpy as np

import attack_oracle as AT
import tailored_attack_oracle as TA

F32_MAX = float(np.finfo(np.float32).max)
STATE_ATTACKS = ("dissensus", "mimic")


def _sum(x, dt):
    """A sum over the parameters; not finite or beyond the fp32 range: +inf."""
    with np.errstate(over="ignore", invalid="ignore"):
        s = dt(np.sum(x, dtype=dt))
    return s if np.isfinite(s) and abs(s) <= F32_MAX else dt(np.inf)


# ------------------------------------------------------------------------------------------------ dissensus
def dissensus(x, V, n_byz, eps):
    """The dissensus message against the receiver's own message x [P] and its honest rows V [n, P]:
    x - (eps / n_byz) * sum_k (v_k - x), summed in row order from 0; eps = 0 gives x."""
    x = np.asarray(x)
    dt = x.dtype.type
    if not (np.isfinite(eps) and eps >= 0) or not 1 <= n_byz <= 16:
        raise ValueError("dissensus needs eps >= 0 and 1 <= n_byz <= 16")
    delta = np.zeros_like(x)
    for v in np.asarray(V, x.dtype):
        delta = delta + (v - x)
    c = dt(dt(eps) / dt(n_byz))
    return x.copy() if c == 0 else (x - c * delta).astype(x.dtype)


# ------------------------------------------------------------------------------------------------ mimic
def centred(V):
    V = np.asarray(V)
    return V - AT.moments(V)[0]


def init_scores(V):
    """e_k = sum_p c_k,p^2 of the centred honest rows (+inf where not finite)."""
    C = centred(V)
    dt = C.dtype.type
    return np.array([_sum(c * c, dt) for c in C], C.dtype)


def init_margin(V):
    """Relative gap between the largest e_k and the largest e_l of a row that differs from it (inf if none)."""
    V = np.asarray(V)
    e = init_scores(V).astype(np.float64)
    k0 = int(np.argmax(e))
    rest = [e[l] for l in range(len(e)) if not np.array_equal(V[l], V[k0])]
    if not rest or not np.isfinite(e[k0]) or e[k0] <= 0:
        return np.inf
    return (e[k0] - max(rest)) / e[k0]


def mimic(V, candidates, z, update, k0=None):
    """(k*, z after the call, t [n] with -inf off the candidates) of the mimic attack over the honest rows V [n, P]
    with direction state z [P] (all zero: not initialised) and update 0 / 1.  k0, when given, replaces the Init choice
    (to follow the kernel through a near tie of e)."""
    V = np.asarray(V)
    dt = V.dtype.type
    C = centred(V)
    z = np.asarray(z, V.dtype).copy()
    cand = sorted(set(candidates))
    if not cand or cand[0] < 0 or cand[-1] >= len(V) or update not in (0, 1):
        raise ValueError("bad candidates or update")
    if not z.any():
        e = init_scores(V)
        if k0 is None:
            k0 = int(np.argmax(e))                          # the first maximum: ties to the smaller k
        if e[k0] > 0 and np.isfinite(e[k0]):
            z = (C[k0] / np.sqrt(e[k0])).astype(V.dtype)
    if update == 1 and z.any():
        s = np.array([_sum(c * z, dt) for c in C], V.dtype)
        u = np.zeros_like(z)
        with np.errstate(over="ignore", invalid="ignore"):
            for k in range(len(C)):
                u = u + s[k] * C[k]
        q = _sum(u * u, dt)
        if q > 0 and np.isfinite(q):
            z = (u / np.sqrt(q)).astype(V.dtype)
    t = np.full(len(V), -np.inf, V.dtype)
    if not z.any():
        return cand[0], z, t
    for k in cand:
        with np.errstate(over="ignore", invalid="ignore"):
            tk = dt(np.sum(C[k] * z, dtype=dt))
        t[k] = tk if np.isfinite(tk) and abs(tk) <= F32_MAX else -np.inf
    best = max(cand, key=lambda k: (t[k], -k))
    return (cand[0] if t[best] == -np.inf else best), z, t


def pick_margin(V, t):
    """Relative gap between the best score and the best score of a candidate row that differs from the best one (inf
    if none): identical rows tie exactly in any precision and go to the smaller index in both."""
    V = np.asarray(V)
    t = np.asarray(t, np.float64)
    best = int(np.argmax(t))
    rest = [t[k] for k in range(len(t)) if np.isfinite(t[k]) and not np.array_equal(V[k], V[best])]
    if not np.isfinite(t[best]) or not rest:
        return np.inf
    return (t[best] - max(rest)) / max(abs(t[best]), 1e-300)


def candidates(j, honest):
    """The trainer's candidates: the entries of S_j that are not the receiver j, unless that leaves none."""
    return [k for k, i in enumerate(honest) if i != j] or list(range(len(honest)))


# ------------------------------------------------------------------------------------------------ update rounds
class StateHook:
    """messages_hook of update_round for attacks of every kind: attacks[b] = (name, param) with a name of
    tailored_attack_oracle.make_hook's or "dissensus" / "mimic"; rules[j] and H[j] as there.  One call is one epoch;
    z[(b, j)] = [critic z, TR z] and steps[(b, j)] carry over between calls (and rounds).  targets[(b, j)] receives
    [critic, TR] agent copied in the last call, and margins[(b, j)] the pick margins.  follow[epoch][(b, j)] (e.g.
    Trainer.mimic_targets() of a run whose last epoch is that one), when given, supplies the pick where the oracle's
    margin is at most `gap`: there a near tie may fall either way in fp32, and the oracle follows the kernel."""

    def __init__(self, labels, in_nodes, attacks, rules, H, seed=0, round_=0, gap=1e-4):
        self.labels, self.in_nodes, self.attacks = labels, in_nodes, attacks
        self.pairs = AT.byzantine_pairs(labels, in_nodes)
        inner_att = {b: (("alie", 0.0) if a[0] in STATE_ATTACKS else a) for b, a in attacks.items()}
        self.inner = TA.make_hook(labels, in_nodes, inner_att, rules, H, seed=seed, round_=round_)
        self.z, self.steps, self.targets, self.margins = {}, {}, {}, {}
        self.follow, self.gap, self.epoch = None, gap, 0

    def __call__(self, epoch, critic_msgs, TR_msgs):
        dt = critic_msgs[0][0].dtype
        per_c, per_t = self.inner(epoch, critic_msgs, TR_msgs)
        lab = self.labels
        upd = {}
        for b, j, honest in self.pairs:
            name, param = self.attacks[b]
            if name not in STATE_ATTACKS:
                continue
            ms, ks, mg = [], [], []
            for t, (msgs, per) in enumerate(((critic_msgs, per_c), (TR_msgs, per_t))):
                V = np.stack([AT.pack(msgs[i], dt) for i in honest])
                if name == "dissensus":
                    n_byz = sum(lab[i] == "Byzantine" and self.attacks[i][0] == "dissensus" for i in self.in_nodes[j])
                    flat = dissensus(AT.pack(msgs[j], dt), V, n_byz, param)
                else:
                    zs = self.z.setdefault((b, j), [np.zeros(V.shape[1], dt), np.zeros(V.shape[1], dt)])
                    u = upd.setdefault((b, j), int(self.steps.get((b, j), 0) < param))
                    k, zs[t], sc = mimic(V, candidates(j, honest), zs[t], u)
                    m = pick_margin(V, sc)
                    f = (self.follow or {}).get(self.epoch, {}).get((b, j))
                    if m <= self.gap and f is not None:
                        k = honest.index(int(f[t])) if honest[k] != int(f[t]) else k
                    ks.append(honest[k])
                    mg.append(m)
                    flat = V[k].copy()
                ms.append(flat)
                per[j] = [AT.unpack(flat, msgs[b]) if i == b else x for i, x in zip(self.in_nodes[j], per[j])]
            if name == "mimic":
                self.targets[(b, j)], self.margins[(b, j)] = ks, mg
        for key, u in upd.items():
            self.steps[key] = self.steps.get(key, 0) + u
        self.epoch += 1
        return per_c, per_t
