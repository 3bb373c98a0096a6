"""The min-max and min-sum Byzantine messages of include/rcmarl.h (rcmarl_adaptive_attack) in NumPy, in the dtype of the
honest messages (fp32 or fp64): the direction, the per-message sums, the constraint bound c and the closed-form gamma,
returning (message, gamma); and a messages hook for attack_oracle.update_round that crafts both these and the attacks of
rcmarl_attack.

As in the kernel, a squared distance (or ||mu||^2, or a) that is not finite or exceeds the fp32 range counts as +inf in
either dtype."""
import numpy as np

import attack_oracle as AT

KINDS = ("minmax", "minsum")
DEVS = ("uv", "std", "sgn")
ATTACKS = tuple(f"{k}_{d}" for k in KINDS for d in DEVS)
F32_MAX = float(np.finfo(np.float32).max)


def _sum(x, dt):
    """sum of x in index order in dtype dt"""
    s = dt(0)
    for v in x:
        s = dt(s + v)
    return s


def _sq(x, y, dt):
    """sum_p x_p y_p in dt; +inf where not finite or beyond the fp32 range (squared distances and norms only)"""
    with np.errstate(over="ignore", invalid="ignore"):
        s = dt(np.sum(np.asarray(x, dt) * np.asarray(y, dt), dtype=dt))
    return s if np.isfinite(s) and s <= F32_MAX else dt(np.inf)


def direction(mu, sigma, dev):
    dt = mu.dtype.type
    if dev == "uv":
        nrm = np.sqrt(_sq(mu, mu, dt))
        if nrm == 0 or not np.isfinite(nrm):
            return np.zeros_like(mu)
        return -mu / nrm
    if dev == "std":
        return -sigma
    if dev == "sgn":
        return -np.sign(mu).astype(mu.dtype)
    raise ValueError(f"unknown direction {dev!r}")


def root(A, b, e, c):
    """The largest root of A g^2 + 2 b g + e = c in the cancellation-free form of the header; 0 when c - e <= 0."""
    dt = type(A)
    m = dt(c - e)
    if not m > 0:
        return dt(0)
    with np.errstate(over="ignore", invalid="ignore"):
        R = np.sqrt(max(dt(b * b + A * m), dt(0)))
        return dt((-b + R) / A) if b <= 0 else dt(m / (b + R))


def parts(values, attack):
    """(mu, d, a, b [n], e [n], D [n, n]) of the honest messages values [n, P] in values' dtype."""
    v = np.asarray(values)
    dt = v.dtype.type
    kind, dev = attack.split("_")
    if kind not in KINDS:
        raise ValueError(f"unknown attack {attack!r}")
    mu, sigma = AT.moments(v)
    d = direction(mu, sigma, dev).astype(v.dtype)
    n = v.shape[0]
    a = _sq(d, d, dt)
    e = np.array([_sq(mu - v[k], mu - v[k], dt) for k in range(n)], v.dtype)
    with np.errstate(over="ignore", invalid="ignore"):
        b = np.array([np.sum((mu - v[k]) * d, dtype=v.dtype) for k in range(n)], v.dtype)
    D = np.zeros((n, n), v.dtype)
    for k in range(n):
        for l in range(k + 1, n):
            D[k, l] = D[l, k] = _sq(v[k] - v[l], v[k] - v[l], dt)
    return mu, d, a, b, e, D


def bound(D, kind):
    """c: the largest pairwise squared distance (minmax) or the largest sum of squared distances of one honest message
    to the others, summed in index order (minsum)."""
    n = D.shape[0]
    dt = D.dtype.type
    if kind == "minmax":
        return dt(max([D[k, l] for k in range(n) for l in range(k + 1, n)], default=dt(0)))
    return dt(max(_sum([D[k, l] for l in range(n) if l != k], dt) for k in range(n)))


def gamma_of(values, attack):
    mu, d, a, b, e, D = parts(values, attack)
    dt = mu.dtype.type
    kind = attack.split("_")[0]
    c = bound(D, kind)
    if not (a > 0 and np.isfinite(a) and np.isfinite(c) and np.isfinite(b).all() and np.isfinite(e).all()):
        return mu, d, dt(0)
    if kind == "minmax":
        g = max(dt(0), min(root(a, b[k], e[k], c) for k in range(len(b))))
    else:
        g = root(dt(dt(len(b)) * a), _sum(b, dt), _sum(e, dt), c)
    return mu, d, (g if np.isfinite(g) else dt(0))


def craft(values, attack, scale):
    """(message, gamma) of the min-max / min-sum attack `attack` ("minmax_uv", ..., "minsum_sgn") with scale s >= 0
    against the honest messages values [n, P]."""
    if not (np.isfinite(scale) and scale >= 0):
        raise ValueError("the scale must be finite and >= 0")
    mu, d, g = gamma_of(values, attack)
    dt = mu.dtype.type
    t = dt(dt(scale) * g)
    return (mu.copy() if t == 0 else (mu + t * d).astype(mu.dtype)), g


def constraint(values, attack, m):
    """(the constrained quantity at the message m, its bound c): max_k ||m - v_k||^2 (minmax) or sum_k ||m - v_k||^2
    (minsum), against c."""
    v = np.asarray(values)
    kind = attack.split("_")[0]
    dist = [float(np.sum((m - v[k]) ** 2)) for k in range(v.shape[0])]
    D = parts(v, attack)[5]
    return (max(dist) if kind == "minmax" else float(np.sum(dist))), float(bound(D, kind))


def make_hook(labels, in_nodes, attacks, seed=0, round_=0, gammas=None):
    """attack_oracle.make_hook for attacks of both kinds: attacks[b] = (name, param) with a name of rcmarl_attack or of
    ATTACKS.  gammas (a dict, optional) receives {(b, j): [critic gamma, TR gamma]} of the last epoch hooked."""
    pairs = AT.byzantine_pairs(labels, in_nodes)

    def hook(epoch, critic_msgs, TR_msgs):
        dt = critic_msgs[0][0].dtype
        per_c = {j: [critic_msgs[i] for i in in_nodes[j]] for j in range(len(labels))}
        per_t = {j: [TR_msgs[i] for i in in_nodes[j]] for j in range(len(labels))}
        for b, j, honest in pairs:
            kind, param = attacks[b]
            gs = []
            for msgs, per in ((critic_msgs, per_c), (TR_msgs, per_t)):
                vals = np.stack([AT.pack(msgs[k], dt) for k in honest])
                if kind in ATTACKS:
                    flat, g = craft(vals, kind, param)
                    gs.append(float(g))
                else:
                    xi = AT.gauss_xi(vals.shape[1], seed, b, j, round_, epoch, dt) if kind == "gauss" else None
                    flat = AT.craft(vals, kind, param, xi)
                m = AT.unpack(flat, msgs[b])
                per[j] = [m if i == b else x for i, x in zip(in_nodes[j], per[j])]
            if gs and gammas is not None:
                gammas[(b, j)] = gs
        return per_c, per_t
    return hook
