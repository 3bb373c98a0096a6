"""The random streams of rcmarl_rollout's Philox branch, restated from include/rcmarl.h (not from the kernel), and the
pieces that let the fp64 oracle (oracle/rpbcac_oracle.py) follow the Trainer's default training loop round by round:

  rollout_draws          the reset positions and action uniforms a Philox-mode launch draws, in the layout of the
                         injected branch and of O.rollout_block;
  reset_counters / action_counters
                         their Philox counters (also used to check that the streams never share a counter);
  default_perm_source    the Trainer's own mini-batch shuffles (perm_source=None);
  oracle_agents_from_trainer / trainer_rows
                         oracle agents and buffer rows read back from a Trainer;
  oracle_rollout / check_rows
                         the oracle's rollout of a block on restated draws, and the exact row comparison with ties
                         excluded;
  round_perms / reassociated / perturbed / with_kernel_adam / yardstick_rounds / yardstick_ratios / yardstick /
  parallel_map           the fp32-spread yardstick of whole update rounds at the reference hyper-parameters, with its
                         conditioning term s_cond.

Philox4x32-10 itself is attack_oracle.philox4x32_10 (integer-exact, checked against the Random123 known answers)."""
import copy
import os
from collections import namedtuple
from concurrent.futures import ProcessPoolExecutor
import multiprocessing

import numpy as np

from attack_oracle import philox4x32_10
from oracle import rpbcac_oracle as O

M32 = 0xFFFFFFFF
RESET_BIT = 0x80000000                     # word 1 of every reset counter
ATTACK_BIT = 0x40000000                    # word 1 of every rcmarl_attack counter (bit 31 clear)
U01 = np.float32(2.0 ** -24)


def _key(seed):
    seed = int(seed)
    return seed & M32, (seed >> 32) & M32


def _env_words(env_offset, n_envs):
    g = int(env_offset) + np.arange(n_envs, dtype=np.uint64)
    return g & np.uint64(M32), g >> np.uint64(32)


def _episode_words(episode_offset, n_episodes):
    return (int(episode_offset) + np.arange(n_episodes, dtype=np.uint64)) & np.uint64(M32)


def reset_counters(*, env_offset, n_envs, episode_offset, n_episodes, n_active):
    """Counter words of the reset draws, each [n_episodes][n_envs][n_active]:
    (g low, g high ^ 0x80000000, episode word, agent) with g = env_offset + env."""
    lo, hi = _env_words(env_offset, n_envs)
    ep = _episode_words(episode_offset, n_episodes)
    shape = (n_episodes, n_envs, n_active)
    return [np.broadcast_to(lo[None, :, None], shape), np.broadcast_to((hi ^ np.uint64(RESET_BIT))[None, :, None], shape),
            np.broadcast_to(ep[:, None, None], shape), np.broadcast_to(np.arange(n_active, dtype=np.uint64), shape)]


def action_counters(*, env_offset, n_envs, episode_offset, n_episodes, max_ep_len, n_slots, n_active):
    """Counter words of the action draws, each [n_episodes][max_ep_len][n_envs][n_active]:
    (g low, g high, episode word, step * n_slots + agent); n_slots is the kernel instantiation (5 or 16)."""
    lo, hi = _env_words(env_offset, n_envs)
    ep = _episode_words(episode_offset, n_episodes)
    shape = (n_episodes, max_ep_len, n_envs, n_active)
    w3 = np.arange(max_ep_len, dtype=np.uint64)[:, None] * np.uint64(n_slots) + np.arange(n_active, dtype=np.uint64)
    return [np.broadcast_to(lo[None, None, :, None], shape), np.broadcast_to(hi[None, None, :, None], shape),
            np.broadcast_to(ep[:, None, None, None], shape), np.broadcast_to(w3[None, :, None, :], shape)]


def u01(w):
    """(w >> 8) * 2^-24: 24 random bits, exact in fp32, in [0, 1)."""
    return (np.asarray(w, np.uint32) >> np.uint32(8)).astype(np.float32) * U01


def rollout_draws(seed, *, env_offset, n_envs, episode_offset, n_episodes, max_ep_len, n_slots, n_active, nrow, ncol):
    """What a Philox-mode rcmarl_rollout draws: (init_states int32 [n_ep][N][n_active][2],
    uniforms float32 [n_ep][L][N][n_active][3]), exactly the arrays its injected branch and O.rollout_block take.
    Resets: px = umulhi(x, nrow), py = umulhi(y, ncol); actions: u0, u1, u2 = u01(x), u01(y), u01(z)."""
    key = _key(seed)
    init = np.empty((n_episodes, n_envs, n_active, 2), np.int32)
    uni = np.empty((n_episodes, max_ep_len, n_envs, n_active, 3), np.float32)
    for e in range(n_episodes):                         # one episode at a time bounds the uint64 temporaries
        kw = dict(env_offset=env_offset, n_envs=n_envs, episode_offset=int(episode_offset) + e, n_episodes=1)
        x, y, _, _ = philox4x32_10(reset_counters(n_active=n_active, **kw), key)
        init[e, ..., 0] = (x[0].astype(np.uint64) * np.uint64(nrow)) >> np.uint64(32)
        init[e, ..., 1] = (y[0].astype(np.uint64) * np.uint64(ncol)) >> np.uint64(32)
        x, y, z, _ = philox4x32_10(action_counters(max_ep_len=max_ep_len, n_slots=n_slots, n_active=n_active, **kw), key)
        uni[e, ..., 0], uni[e, ..., 1], uni[e, ..., 2] = u01(x[0]), u01(y[0]), u01(z[0])
    return init, uni


def default_perm_source(seed):
    """The Trainer's shuffles with perm_source=None: torch.randperm(T, int32) from a CPU generator seeded
    seed * 7919 + 17, called in the Trainer's draw order (which is the oracle's)."""
    import torch
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed) * 7919 + 17)
    return lambda T: torch.randperm(T, generator=g, dtype=torch.int32).numpy()


def oracle_agents_from_trainer(tr, dtype=np.float64):
    """Oracle agents holding the Trainer's current state (tr.state_dict()): actor / critic / TR weights, the Malicious
    agents' critic_local, and the Keras-Adam m, v, t of every actor, with the Trainer's per-agent H, fast_lr, slow_lr."""
    from rcmarl import nets
    sd = tr.state_dict(include_buffer=False)
    n, NA = tr.n_real, tr.NA

    def net(name, i, f, n_out):
        return nets.unpack_padded(sd[name][i].numpy(), f * n, f * NA, n_out)
    agents = []
    for i in range(n):
        lab = tr.labels[i]
        a, c, t = net("actor", i, 2, 5), net("critic", i, 2, 1), net("tr", i, 3, 1)
        if lab == "Cooperative":
            ag = O.RPBCACOracleAgent(a, c, t, tr.slow_lr[i], tr.fast_lr[i], tr.gamma, H=tr.H[i], dtype=dtype)
        elif lab == "Malicious":
            ag = O.MaliciousOracleAgent(a, c, t, tr.slow_lr[i], tr.fast_lr[i], tr.gamma,
                                        critic_local_w=net("critic_local", i, 2, 1), dtype=dtype)
        elif lab == "Greedy":
            ag = O.GreedyOracleAgent(a, c, t, tr.slow_lr[i], tr.fast_lr[i], tr.gamma, dtype=dtype)
        elif lab == "Faulty":
            ag = O.FaultyOracleAgent(a, c, t, tr.slow_lr[i], tr.gamma, dtype=dtype)
        else:
            raise ValueError(f"no oracle agent for label {lab!r}")
        steps = int(sd["adam_t"][i])
        if steps:
            ag.adam.m = [x.astype(dtype) for x in net("adam_m", i, 2, 5)]
            ag.adam.v = [x.astype(dtype) for x in net("adam_v", i, 2, 5)]
            ag.adam.t = steps
        agents.append(ag)
    return agents


def trainer_rows(tr, t0, t1):
    """Time rows [t0, t1) of the Trainer's buffer for its real agents as float32 arrays in the oracle's layout:
    s, ns (B, n, 2) and a, r (B, n, 1), B = (t1 - t0) * n_envs."""
    n, NA, N = tr.n_real, tr.NA, tr.N
    lo, hi = t0 * N, t1 * N
    sa = tr.sa[lo:hi].view(-1, NA, 3)[:, :n].cpu().numpy()
    ns = tr.ns[lo:hi].view(-1, NA, 2)[:, :n].cpu().numpy()
    r = tr.r[lo:hi].view(-1, NA, 1)[:, :n].cpu().numpy()
    return sa[:, :, :2].copy(), ns, sa[:, :, 2:].copy(), r


def oracle_rollout(agents, desired, nrow, ncol, draws, gamma, mu=0.1, scaling=True):
    """O.rollout_block on the restated draws; every agent logs est (the kernel computes it for all agents)."""
    init, U = draws
    n_ep, L_, N, n = U.shape[:4]
    env = O.GridWorldOracle(nrow, ncol, n, desired, n_envs=N, scaling=scaling)
    S, NS, A, Rw, est, ret = O.rollout_block(env, agents, ["Cooperative"] * n, n_episodes=n_ep, max_ep_len=L_,
                                             gamma=gamma, init_states=init, uniforms=U, mu=mu)
    return (S, NS, A, Rw), est, ret


def check_rows(got, want, n_ep, L_, N):
    """got / want: (s, ns, a, r) of n_ep episodes x L_ steps x N environments.  -> ok[n_ep, N]: episodes free of ties,
    whose rows must then be exactly the oracle's."""
    act_equal = got[2][..., 0] == want[2][..., 0]
    assert act_equal.mean() > 0.999, act_equal.mean()
    ok = np.ones((n_ep, N), bool)
    for row, _ in np.argwhere(~act_equal):
        t, e = divmod(row, N)
        ok[t // L_, e] = False
    assert ok.mean() > 0.9, ok.mean()
    mask = np.repeat(ok, L_, axis=0).reshape(-1)
    for g, w, name in zip(got, want, ("s", "ns", "a", "r")):
        assert np.array_equal(g[mask], np.asarray(w, np.float32)[mask]), name
    return ok


# ------------------------------------------------------------------------------------------ the fp32-spread yardstick
# Measured on an H100 (the cases of test_reference_scale_gpu.py): ||gpu - o64|| / s up to 5.5 normwise and 7.1 in the
# max norm over weights and Adam slots; c = 4 failed on those.
YARD_C = 8.0            # ||gpu - o64|| may be this many times the fp32 spread s ...
YARD_C_INF = 12.0       # ... (max |gpu - o64| this many times s_inf) ...
YARD_FLOOR = 1e-6       # ... or of YARD_FLOOR x ||o64||, whichever is larger


def round_perms(perm_source, labels, T, *, n_epochs, n_actor_steps):
    """The time-row permutations one O.update_round draws from perm_source, in its draw order: per epoch 20 per Greedy
    and 30 per Malicious agent (10 per mini-batch fit), then one actor window's per non-cooperative agent."""
    n_fit = n_epochs * sum({"Greedy": 20, "Malicious": 30}.get(lab, 0) for lab in labels)
    n_act = sum(lab != "Cooperative" for lab in labels)
    return [np.asarray(perm_source(T)) for _ in range(n_fit)] + \
        [np.asarray(perm_source(min(n_actor_steps, T))) for _ in range(n_act)]


def reassociated(buf, perms, *, n_envs, n_actor_steps, n_act, mb_times=32, actor_mb_times=200, order="reversed"):
    """The same update round with another summation order: the buffer's time rows moved inside the part before the
    actor window and inside the window, its environments moved inside every time row, and the permutations mapped
    so that each mini-batch holds the same rows, moved likewise.  order "reversed" reverses each of these sequences;
    "rotated" rotates each by half its length (a third order, which differs from the first two at n_envs = 1 too).
    The last n_act permutations are the actor windows'.  Every sum sees the same terms, so only the rounding changes."""
    move = {"reversed": lambda x: x[::-1], "rotated": lambda x: np.roll(x, len(x) // 2)}[order]
    N = n_envs
    T = buf[0].shape[0] // N
    Ta = min(n_actor_steps, T)
    rho = np.concatenate([move(np.arange(T - Ta)), T - Ta + move(np.arange(Ta))])    # new time row j holds old row rho[j]
    inv = np.argsort(rho)
    rows = (rho[:, None] * N + move(np.arange(N))[None, :]).reshape(-1)

    def moved(p, mb):
        q = np.array(p)
        for k in range(0, len(q), mb):
            q[k:k + mb] = move(q[k:k + mb]).copy()
        return q
    n_fit = len(perms) - n_act
    return (tuple(np.ascontiguousarray(x[rows]) for x in buf),
            [moved(inv[p], mb_times) for p in perms[:n_fit]] +
            [moved(inv[T - Ta + np.asarray(p)] - (T - Ta), actor_mb_times) for p in perms[n_fit:]])


def perturbed(agents, rs):
    """Copies of agents whose every weight and Adam slot is multiplied element-wise by 1 + d, d uniform in +-2^-24 from
    rs (a RandomState): the error of merely storing the round's starting point in fp32."""
    out = copy.deepcopy(agents)
    u = 2.0 ** -24

    def scale(arrays):
        for k, x in enumerate(arrays):
            arrays[k] = x * (1.0 + rs.uniform(-u, u, np.shape(x))).astype(x.dtype)
    for ag in out:
        for net in ag.get_parameters():
            scale(net)
        if ag.adam.m is not None:
            scale(ag.adam.m)
            scale(ag.adam.v)
    return out


def with_kernel_adam(agents):
    """agents whose Keras Adam uses the kernel's float32 constants (O.KerasAdam fp32_betas): rcmarl_adam_apply forms
    1 - 0.999 as 1.f - 0.999f, 1.3e-5 below 0.001, which puts every Adam v 1.3e-5 relative away from the exact
    constant's -- a fixed difference of the formula, not rounding, so the yardstick's oracle rounds use it."""
    for ag in agents:
        ag.adam.fp32_betas = True
    return agents

def _oracle_round(agents, labels, in_nodes, buf, perms, kw):
    left = list(perms)

    def source(T):
        p = left.pop(0)
        assert len(p) == T
        return p
    loss = O.update_round(agents, labels, in_nodes, *buf, perm_source=source, **kw)
    assert not left
    return agents, loss


def yardstick_jobs(r, n_cond=0):
    """The _oracle_round jobs of one update round r (see yardstick_rounds): fp64, fp32, fp32 on reassociated(...), then
    n_cond fp64 rounds from perturbed(a64) (RandomState(24), in sequence, so a smaller n_cond is a prefix of a larger
    one's) on the same buffer and permutations."""
    kw = r["kw"]
    n_act = sum(lab != "Cooperative" for lab in r["labels"])
    alt_buf, alt_perms = reassociated(r["buf"], r["perms"], n_envs=kw["n_envs"], n_actor_steps=kw["n_actor_steps"],
                                      n_act=n_act)
    rs = np.random.RandomState(24)
    return [(r["a64"], r["labels"], r["in_nodes"], r["buf"], r["perms"], kw),
            (r["a32"], r["labels"], r["in_nodes"], r["buf"], r["perms"], kw),
            (r["a32b"], r["labels"], r["in_nodes"], alt_buf, alt_perms, kw)] + \
        [(perturbed(r["a64"], rs), r["labels"], r["in_nodes"], r["buf"], r["perms"], kw) for _ in range(n_cond)]


def yardstick_rounds(rounds, *, n_cond=0, workers=None):
    """rounds: one dict per update round with the oracle agents at the Trainer's state before it in fp64 ("a64") and
    twice in fp32 ("a32", "a32b"), labels, in_nodes, the Trainer's buffer rows ("buf"), the permutations the Trainer
    drew ("perms", round_perms) and the O.update_round keywords ("kw").  Runs the oracle rounds of every entry
    (yardstick_jobs): fp64, fp32, fp32 reassociated, and n_cond perturbed fp64 rounds for the conditioning term.  They
    are independent, so they run in parallel worker processes.  Returns per round [(agents, losses)] in that order."""
    jobs = [job for r in rounds for job in yardstick_jobs(r, n_cond)]
    out = parallel_map(_oracle_round, jobs, workers)
    per = 3 + n_cond
    return [out[per * k:per * k + per] for k in range(len(rounds))]


def parallel_map(fn, jobs, workers=None):
    """[fn(*args) for args in jobs] in spawned worker processes, each with one BLAS thread (the oracle's matrices are
    small; the jobs, not the threads, fill the cores)."""
    names = ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS")
    saved = {k: os.environ.get(k) for k in names}
    os.environ.update({k: "1" for k in names})
    try:
        with ProcessPoolExecutor(workers or min(len(jobs), os.cpu_count() or 1),
                                 mp_context=multiprocessing.get_context("spawn")) as ex:
            return list(ex.map(fn, *zip(*jobs)))
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def round_tensors(agents):
    """name -> array of the state an update round leaves: every agent's nets (actor, critic, TR, critic_local) and its
    Keras-Adam m and v."""
    out = {}
    for i, ag in enumerate(agents):
        for n, net in enumerate(ag.get_parameters()):
            for k, x in enumerate(net):
                out[f"agent {i} net {n} array {k}"] = x
        for k in range(6):
            out[f"agent {i} adam_m {k}"] = ag.adam.m[k]
            out[f"agent {i} adam_v {k}"] = ag.adam.v[k]
    return out


Ratio = namedtuple("Ratio", "name norm inf excess cond_over_s o32_agree rel s_rel cond_rel")


def yardstick_ratios(got, o64, o32s, cond=(), *, c=YARD_C, c_inf=YARD_C_INF, floor=YARD_FLOOR):
    """Per tensor of o64 a Ratio: norm = ||got - o64|| / tol and inf = max |got - o64| / tol_inf with the yardstick's
    tol = max(s, s_cond, floor ||o64||) (and its max-norm twin), excess = max(norm / c, inf / c_inf) (the tensor passes
    when excess <= 1), cond_over_s = s_cond / s, o32_agree = ||o32 - o32b|| / s, and rel, s_rel, cond_rel =
    ||got - o64||, s, s_cond over ||o64||."""
    rows = []
    for name, x in o64.items():
        x = np.asarray(x, np.float64)
        g = np.asarray(got[name], np.float64)
        d = [np.asarray(o[name], np.float64) - x for o in o32s]
        dc = [np.asarray(o[name], np.float64) - x for o in cond]
        s, s_inf = max(np.linalg.norm(e) for e in d), max(np.abs(e).max() for e in d)
        sc, sc_inf = max([np.linalg.norm(e) for e in dc], default=0.0), max([np.abs(e).max() for e in dc], default=0.0)
        tol, tol_inf = max(s, sc, floor * np.linalg.norm(x)), max(s_inf, sc_inf, floor * np.abs(x).max())
        err, err_inf = np.linalg.norm(g - x), np.abs(g - x).max()
        norm, inf = err / tol if tol > 0 else 0.0, err_inf / tol_inf if tol_inf > 0 else 0.0
        if tol == 0 and err > 0:
            norm = inf = np.inf
        rows.append(Ratio(name, norm, inf, max(norm / c, inf / c_inf), sc / s if s > 0 else (np.inf if sc > 0 else 0.0),
                          np.linalg.norm(d[0] - d[1]) / s if s > 0 else 0.0,
                          *(v / max(np.linalg.norm(x), 1e-300) for v in (err, s, sc))))
    return rows


def yardstick(got, o64, o32s, cond=(), *, c=YARD_C, c_inf=YARD_C_INF, floor=YARD_FLOOR, msg=""):
    """The fp32-spread yardstick.  For every tensor x of an update round (round_tensors: weights, Adam m and v), with
    o64 the fp64 oracle's, o32s the fp32 oracle's in two summation orders and cond the fp64 oracle's from perturbed
    starting points (yardstick_rounds):

        s      = max over the fp32 runs of ||o32 - o64||         (Frobenius norm)
        s_cond = max over the perturbed fp64 runs of ||oc - o64||
        ||got - o64||       <= c x max(s, s_cond, floor x ||o64||)
        max |got - o64|     <= c_inf x max(s_inf, s_cond_inf, floor x max |o64|)   (the same, element-wise)

    At 10 epochs a fixed element-wise tolerance does not work: an fp32 restatement of the same maths already misses
    fp64 by several times DESIGN.md's whole-round tolerance on some seeds: ten epochs of consensus and projection
    carry rounding forward, and a mini-batch fit can meet a leaky-ReLU sign flip (yardstick_team).  s is the rounding error of fp32 arithmetic on these very inputs, so a kernel must
    stay within a few times of it.  Two fp32 samples do not show how far rounding *can* move an ill-conditioned
    tensor, though: s_cond samples (condition number x fp32 unit round-off) for that tensor on those inputs, as the
    movement of the exact round under the error of storing its starting point in fp32.  Where the round is well
    conditioned s_cond is at or below s and changes nothing; with cond = () the bound is the two-sample one.
    (A scalar such as a loss gives s from a single error sample, too noisy for this; losses keep the whole-round
    tolerance.)

    Measured with the CPU oracle at N = 1, T = 1000 (tests/test_yardstick_cpu.py): the largest s_cond / ||o64|| over
    all tensors is 4.4e-7, 5.5e-7, 5.5e-7 for K = 2, 4, 8 perturbed rounds on M16 and 3.1e-7 for all three on C2, so
    K = 4 is enough, and s_cond exceeds max(s, floor ||o64||) on no tensor of C2, Greedy + Faulty or M16: the fp64
    round is well conditioned to first order everywhere, M16 included.  The term is therefore used for that
    measurement only (cond = () elsewhere).  What makes M16's round hard is leaky-ReLU sign flips in the adversaries'
    mini-batch fits (yardstick_team), which s_cond does not sample.

    Prints the largest ||got - o64|| / tol and max-norm ratio, the median over the tensors of ||o32 - o32b|| / s (it
    tells rounding, about 1, from a systematic fp32 / fp64 difference, much less than 1) and the largest s_cond / s
    with its tensor; returns the Ratios (yardstick_ratios)."""
    rows = yardstick_ratios(got, o64, o32s, cond, c=c, c_inf=c_inf, floor=floor)
    worst = max(rows, key=lambda row: row.norm)
    wc = max(rows, key=lambda row: row.cond_over_s)
    print(f"\n{msg}: largest ||gpu - o64|| / tol = {worst.norm:.2f} ({worst.name}); largest max-norm ratio "
          f"{max(row.inf for row in rows):.2f}; median ||o32 - o32b|| / s = {np.median([row.o32_agree for row in rows]):.2f}"
          f"; largest s_cond / s = {wc.cond_over_s:.2f} ({wc.name})")
    for row in sorted(rows, key=lambda row: -row.excess)[:4]:
        print(f"    {row.name}: {row.norm:.2f} / max-norm {row.inf:.2f}, ||gpu - o64|| / ||o64|| = {row.rel:.1e}, "
              f"s_cond / s = {row.cond_over_s:.2f}")
    bad = [f"{row.name}: ||gpu - o64|| is {row.norm:.2f} x tol (limit {c}), max norm {row.inf:.2f} x (limit {c_inf})"
           for row in rows if not row.excess <= 1]
    assert not bad, f"{msg}: " + "; ".join(bad)
    return rows


FLIP_REL = 5e-2         # a tensor excused by yardstick_team may still miss fp64 by no more than this share of its norm


def yardstick_team(got, o64, o32s, cond=(), *, labels, in_nodes, max_flips, msg="", **kw):
    """The yardstick for teams whose adversaries' mini-batch fits meet leaky-ReLU sign flips.  An fp32 fit whose hidden
    pre-activation on some row lies within rounding of zero takes slope 1 in one summation order and 0.1 in another;
    that one SGD step moves the net by about 1e-4 of its norm, later flips follow, and after ten epochs the net is 1e-3
    to 2e-2 away from the fp64 fit while the orders that define s may have met no flip (measured in
    tests/test_yardstick_cpu.py).  Such an event is correct arithmetic, it is confined to the fitted agent and to the
    cooperative agents that receive its messages, and it is rare per agent and round.  So every tensor must pass
    yardstick_ratios except those of at most max_flips Malicious or Greedy agents and of cooperative agents that have
    one of these among their in-neighbours, and an excused tensor must still be within FLIP_REL of ||o64||.  A fault
    that reaches more adversaries, a cooperative agent with no flipped in-neighbour, or the Faulty agent fails.
    Prints the ratios over the tensors held and the agents excused; returns (Ratios, flipped agents)."""
    rows = yardstick_ratios(got, o64, o32s, cond, **kw)
    agent = lambda row: int(row.name.split()[1])                                   # noqa: E731
    bad = [row for row in rows if not row.excess <= 1]
    bad_agents = {agent(row) for row in bad}
    flipped = sorted(i for i in bad_agents if labels[i] in ("Malicious", "Greedy"))
    downstream = sorted(i for i in bad_agents - set(flipped) if labels[i] == "Cooperative" and set(in_nodes[i]) & set(flipped))
    stray = sorted(bad_agents - set(flipped) - set(downstream))
    held = [row for row in rows if agent(row) not in bad_agents]
    worst = max(held, key=lambda row: row.excess)
    print(f"\n{msg}: {len(rows) - len(bad)} of {len(rows)} tensors within the bound; over the agents without a miss the "
          f"largest ||gpu - o64|| / tol = {max(r.norm for r in held):.2f}, max-norm ratio {max(r.inf for r in held):.2f} "
          f"({worst.name}); flipped adversaries {flipped}, cooperative agents downstream of them {downstream}"
          + (f"; largest miss {max(r.excess for r in bad):.0f} x the bound, {max(r.rel for r in bad):.1e} of the norm "
             f"({max(bad, key=lambda r: r.excess).name})" if bad else ""))
    assert not stray, f"{msg}: agents {stray} miss the bound with no flipped adversary among their in-neighbours: " + \
        "; ".join(f"{r.name} {r.excess:.1f} x" for r in bad if agent(r) in stray)[:600]
    assert len(flipped) <= max_flips, f"{msg}: adversaries {flipped} miss the bound, more than {max_flips} sign-flip events"
    far = [r for r in bad if not r.rel <= FLIP_REL]
    assert not far, f"{msg}: beyond {FLIP_REL} of the norm: " + "; ".join(f"{r.name} {r.rel:.1e}" for r in far)[:600]
    return rows, flipped
