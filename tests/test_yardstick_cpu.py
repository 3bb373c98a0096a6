"""What the fp32-spread yardstick (rollout_oracle.yardstick) accepts and what it rejects, measured without a GPU.

test_reference_scale_gpu.py judges the kernels' ten-epoch update rounds by that yardstick alone, so this file judges
the yardstick.  Update rounds are built entirely from the oracle at the reference hyper-parameters (bench.HYPER: 10
epochs, blocks of 50 episodes x 20 steps) and the smallest shapes that keep the structure, N = 1 and T = 1000:

  C2             4 cooperative agents + 1 Malicious (three mini-batch chains), H = 1;
  greedy_faulty  3 cooperative agents + Greedy + Faulty with common_reward;
  M16            the 16-agent team (16 chains, per-agent H and fast_lr), whose adversaries' fits meet sign flips.

The rows are the oracle's rollout (oracle_rollout) of the kernel's Philox draws (rollout_draws), rounded to fp32 as the
Trainer's buffer holds them; the shuffles are the Trainer's (default_perm_source / round_perms).  The round starts
from the team's weights after one single-epoch warm-up round on the same rows, rounded to fp32, so that every agent
has Keras-Adam moments and a step count as in any round but the first.

"The kernel" is played by an fp32 oracle round in a third summation order (reassociated(order="rotated"): time rows
and mini-batch contents rotated by half), distinct from the two orders that define s.  It must pass the yardstick as
it stands, and fail it, on the tensors the fault reaches, once one input is made subtly wrong (MUTANTS; no oracle code
is patched).  One mutant is a negative control: a buffer reward moved by 1 ulp is rounding, and must still pass.
All rounds of all cases are independent and run in one pool of worker processes.

Measured with the CPU oracle (NumPy / OpenBLAS on 8 x86-64 cores; nothing here runs on a GPU), n_cond = 4, as the
excess = max(||got - o64|| / (8 tol), max |got - o64| / (12 tol_inf)) on the worst tensor the fault reaches (above 1
the yardstick rejects), `pytest tests/test_yardstick_cpu.py -q -s`, 45 s for the 51 oracle rounds (only tensors on which the round without the
fault passes count):

                           C2        greedy_faulty   M16
  third order, no fault    0.19      0.28            0.80 on cooperative agents; 944 on two Malicious agents
  fast_lr x (1 + 1e-3)     14        124             306
  gamma 0.9 -> 0.9001      43        137             2674
  H - 1                    1261      23836           2324
  in-neighbour dropped     4043      1828            4586
  row in the wrong step    24        26              0.50   (not seen)
  tail off by one          1.6       46              0.29   (not seen)
  tail off by one, always  355       201             14
  stale Adam t             114       1134            0.65   (not seen)
  reward + 1 ulp           0.19      0.26            no tensor fails that passed without it

What the table says.  On C2 and Greedy + Faulty correct fp32 arithmetic sits at 0.2 to 0.3 of the bound and every
mutant is rejected but one: a single off-by-one tail in one of 3200 SGD steps on C2 is at 1.6, within the noise of the
fp32 samples (0.2 to 2.5 when the fault is put in other epochs; SGD forgets it rather than compounding it), so that
pair is printed and not asserted (WITHIN_NOISE); the same fault in every epoch, which is what a kernel bug would be, is
rejected at 355.  On M16 the instrument is blind to the three single-step faults on the agent they act on (Malicious
agent 1, whose nets already differ by 1e-3 of their norm between the fp32 samples); they are strict expected failures.

The conditioning term.  The fp64 round moves by at most 5.5e-7 of a tensor's norm under the 2^-24 perturbation (max
over K = 2, 4, 8 perturbed rounds: 4.4e-7, 5.5e-7, 5.5e-7 on M16; 3.1e-7 for all three on C2), so s_cond never exceeds
max(s, floor) and no bound changes: every round here, M16's included, is well conditioned to first order.  The term is
therefore measured here only; test_reference_scale_gpu.py does not use it.

What M16 does instead.  An adversary's net fitted by mini-batch SGD leaves the fp64 round by 1e-3 to 2e-2 of its norm
in some fp32 summation orders and stays within 1e-6 in others: agents 3 and 11 in the two orders that define s, agents
5 and 9 in the third.  Followed alone, agent 9's critic_local agrees with fp64 to 1e-6 in all three orders for six outer
epochs; then in one SGD step (outer epoch 6, inner 0, step 4) the two orders part by 7e-5: on one row of that
mini-batch the pre-activation of hidden unit 2 of the second layer is -3.1e-7 in one order and +1.2e-7 in the other,
so its leaky-ReLU slope is 0.1 in one and 1 in the other.  Further flips follow and the nets are 6e-3 apart by the
tenth epoch.  A 2^-24 perturbation of the fp64 fit moves a pre-activation by about 1e-8 and so meets such a flip ten
to a hundred times less often than fp32 rounding does; none of 8 perturbed rounds met one.  The event is correct
arithmetic, confined to the fitted agent and the cooperative agents that hear it, so yardstick_team excuses a bounded
number of such agents per round and holds everything else; the M16 calibration here and the M16 rounds on the GPU use
it.  On the agents it excuses it holds nothing beyond 5e-2 of the norm, and where s itself contains a flip (agents 3
and 11 here, s up to 2.4e-2 of the norm) the plain bound is that loose: on M16 the yardstick holds 403 of 504 tensors
to better than 1e-4 of their norm after one epoch and 48 to 103 after ten (H100 rounds at N = 2).
"""
import copy
import os
import time

import numpy as np
import pytest

import bench                                          # HYPER only: importing it runs nothing
import rollout_oracle as R
import team_util as T16

f32, f64 = np.float32, np.float64
SEED = 1234
HYPER = bench.HYPER
COND_REL_MAX = 2e-6                                   # s_cond / ||o64|| stays below this (measured: at most 5.5e-7)
N_COND = 4                                            # as test_reference_scale_gpu.py
CASES = ("c2", "greedy_faulty", "M16")
SLOW = {"M16"}
# The M16 rounds (16 per case, each 6.5 s on one core; the whole file takes 35 s on 8 cores with them) run unless RCMARL_YARDSTICK_SKIP_M16 is set.
skip_m16 = pytest.mark.skipif(bool(os.environ.get("RCMARL_YARDSTICK_SKIP_M16")),
                              reason="RCMARL_YARDSTICK_SKIP_M16 is set: the 16-agent oracle rounds are skipped")


def cast_agents(agents, dtype):
    """Copies of oracle agents computing in dtype, their weights and Adam moments rounded to it."""
    out = copy.deepcopy(agents)
    for ag in out:
        ag.dtype = dtype
        for net in ag.get_parameters():
            net[:] = [np.asarray(x, dtype) for x in net]
        if ag.adam.m is not None:
            ag.adam.m = [np.asarray(x, dtype) for x in ag.adam.m]
            ag.adam.v = [np.asarray(x, dtype) for x in ag.adam.v]
    return out


def build_round(name, *, n_epochs=HYPER["n_epochs"], n_episodes=HYPER["n_ep_fixed"], seed=SEED):
    """The update round of team `name` (team_util.loop_team) after its first block at N = 1, as a yardstick_rounds
    entry: rows from the oracle's rollout of the Philox draws, the Trainer's default shuffles, the start state described
    in the module docstring."""
    cfg = {**HYPER, **T16.loop_team(name)}
    labels, n = cfg["labels"], len(cfg["labels"])
    per = lambda v: list(v) if isinstance(v, (list, tuple)) else [v] * n          # noqa: E731
    agents = R.with_kernel_adam(T16.oracle_agents(labels, cfg["weights"], per(cfg["H"]), per(cfg["fast_lr"]),
                                                  cfg["gamma"], cfg["slow_lr"]))
    L_ = cfg["max_ep_len"]
    draws = R.rollout_draws(seed, env_offset=0, n_envs=1, episode_offset=0, n_episodes=n_episodes, max_ep_len=L_,
                            n_slots=5 if n <= 5 else 16, n_active=n, nrow=cfg["nrow"], ncol=cfg["ncol"])
    rows, _, _ = R.oracle_rollout(agents, cfg["desired"], cfg["nrow"], cfg["ncol"], draws, cfg["gamma"])
    buf = tuple(np.asarray(x, f32) for x in rows)
    T = n_episodes * L_
    kw = dict(n_envs=1, n_epochs=n_epochs, n_actor_steps=T, common_reward=cfg.get("common_reward", False))
    source = R.default_perm_source(seed)
    warm = R.round_perms(source, labels, T, n_epochs=1, n_actor_steps=T)
    R._oracle_round(agents, labels, cfg["in_nodes"], buf, warm, {**kw, "n_epochs": 1})
    a32 = cast_agents(agents, f32)
    return dict(T=T, labels=labels, in_nodes=cfg["in_nodes"], buf=buf, kw=kw, a64=cast_agents(a32, f64), a32=a32,
                a32b=copy.deepcopy(a32), perms=R.round_perms(source, labels, T, n_epochs=n_epochs, n_actor_steps=T))


# ------------------------------------------------------------------------------------------------------- the mutants
def _targets(r):
    """(adv, coop, chain, net): the first agent with mini-batch chains, the first cooperative agent whose H can go
    down by one, the index in r["perms"] of the last inner epoch of adv's first chain in the last outer epoch, and the
    net (round_tensors numbering) that chain fits: a Malicious agent's critic_local (3) or a Greedy agent's TR (2)."""
    labels = r["labels"]
    per_agent = [{"Greedy": 20, "Malicious": 30}.get(lab, 0) for lab in labels]
    adv = next(i for i, k in enumerate(per_agent) if k)
    coop = next(i for i, lab in enumerate(labels) if lab == "Cooperative" and r["a32"][i].H >= 1)
    chain = (r["kw"]["n_epochs"] - 1) * sum(per_agent) + sum(per_agent[:adv]) + 9
    return adv, coop, chain, 3 if labels[adv] == "Malicious" else 2


def _chain_tensors(r, adv, net):
    """Where a fault in adv's first chain shows: the net it fits and, for a Malicious agent, the actor and Adam slots
    that critic_local's TD errors drive."""
    own = [f"agent {adv} net {net}"]
    return own + [f"agent {adv} net 0", f"agent {adv} adam_"] if r["labels"][adv] == "Malicious" else own


def _mutate(r, mutant):
    """-> (agents, in_nodes, buf, perms) of the fp32 round with one input made wrong, and the tensor-name prefixes the
    fault must show on (None: it must not show)."""
    adv, coop, chain, net = _targets(r)
    agents, in_nodes = copy.deepcopy(r["a32"]), [list(x) for x in r["in_nodes"]]
    buf, perms = tuple(x.copy() for x in r["buf"]), [np.array(p) for p in r["perms"]]
    mb = 32
    last = (len(perms[chain]) - 1) // mb * mb                        # first entry of the short final mini-batch
    if mutant == "fast_lr":                                          # a mis-scaled learning rate in one agent's chains
        agents[adv].fast_lr *= 1 + 1e-3
        where = [f"agent {adv} net {k}" for k in (1, 2, 3)]
    elif mutant == "gamma":                                          # the wrong discount in every TD target
        for ag in agents:
            ag.gamma = 0.9001
        where = [f"agent {i} net {k}" for i in range(len(agents)) for k in (1, 3)]
    elif mutant == "H":                                              # one agent trims one value too few
        agents[coop].H -= 1
        where = [f"agent {coop} net {k}" for k in (1, 2)]
    elif mutant == "in_node":                                        # one agent misses one neighbour's message
        in_nodes[coop] = in_nodes[coop][:-1]
        where = [f"agent {coop} net {k}" for k in (1, 2)]
    elif mutant == "row_in_wrong_step":                              # two rows swapped across a mini-batch boundary
        p = perms[chain]
        p[last - 1], p[last] = p[last], p[last - 1]
        where = _chain_tensors(r, adv, net)
    elif mutant == "tail_off_by_one":                                # the tail reads one row twice, another never
        perms[chain][-1] = perms[chain][-2]
        where = _chain_tensors(r, adv, net)
    elif mutant == "tail_always":                                    # the same off-by-one in every epoch of the chain
        E = r["kw"]["n_epochs"]
        per_epoch = (len(perms) - sum(lab != "Cooperative" for lab in r["labels"])) // E
        for e in range(E):
            for inner in range(10):
                q = perms[chain - 9 - (E - 1 - e) * per_epoch + inner]
                q[-1] = q[-2]
        where = _chain_tensors(r, adv, net)
    elif mutant == "stale_adam_t":                                   # lr_t of the step before
        agents[adv].adam.t -= 1
        where = [f"agent {adv} net 0", f"agent {adv} adam_"]
    elif mutant == "reward_ulp":                                     # negative control: rounding, not a bug
        t = len(buf[3]) // 2
        buf[3][t, adv, 0] = np.nextafter(buf[3][t, adv, 0], f32(-np.inf))
        where = None
    else:
        raise ValueError(mutant)
    return (agents, in_nodes, buf, perms), where


MUTANTS = ("fast_lr", "gamma", "H", "in_node", "row_in_wrong_step", "tail_off_by_one", "tail_always", "stale_adam_t",
           "reward_ulp")
# (team, mutant) pairs whose excess is within the noise of the fp32 samples (it moves with the BLAS and the core count):
# printed, not asserted
WITHIN_NOISE = {("c2", "tail_off_by_one")}
# (team, mutant) pairs the yardstick cannot see, with the measured excess (1 = at the bound) on the faulted tensors
BLIND = {("M16", "row_in_wrong_step"): "M16 / row_in_wrong_step: 0.50 of the bound on agent 1's critic_local (s is 1e-3 of its norm there)",
         ("M16", "tail_off_by_one"): "M16 / tail_off_by_one: 0.29 of the bound on agent 1's critic_local",
         ("M16", "stale_adam_t"): "M16 / stale_adam_t: 0.65 of the bound on agent 1's actor"}


def _kernel_job(r, agents, in_nodes, buf, perms):
    """The stand-in kernel: the fp32 round in the third summation order."""
    kw = r["kw"]
    n_act = sum(lab != "Cooperative" for lab in r["labels"])
    buf3, perms3 = R.reassociated(buf, perms, n_envs=kw["n_envs"], n_actor_steps=kw["n_actor_steps"], n_act=n_act,
                                  order="rotated")
    return (agents, r["labels"], in_nodes, buf3, perms3, kw)


def run_cases(names, mutants=MUTANTS, n_cond=N_COND):
    """All oracle rounds of the named cases in one pool -> name -> dict(o64, o32s, cond: round_tensors of the
    yardstick's rounds; kernel: of the unmutated stand-in; mutant -> (round_tensors, where))."""
    jobs, plan = [], {}
    for name in names:
        r = build_round(name)
        mine = R.yardstick_jobs(r, n_cond) + [_kernel_job(r, copy.deepcopy(r["a32"]), r["in_nodes"], r["buf"], r["perms"])]
        where = {}
        for m in mutants:
            args, where[m] = _mutate(r, m)
            mine.append(_kernel_job(r, *args))
        plan[name] = (len(jobs), len(mine), where)
        jobs += mine
    out = [R.round_tensors(agents) for agents, _ in R.parallel_map(R._oracle_round, jobs)]
    res = {}
    for name, (lo, cnt, where) in plan.items():
        o = out[lo:lo + cnt]
        res[name] = dict(o64=o[0], o32s=o[1:3], cond=o[3:3 + n_cond], kernel=o[3 + n_cond],
                         **{m: (o[4 + n_cond + k], where[m]) for k, m in enumerate(mutants)})
    return res


@pytest.fixture(scope="module")
def results():
    names = [c for c in CASES if not (c in SLOW and os.environ.get("RCMARL_YARDSTICK_SKIP_M16"))]
    t0 = time.time()
    res = run_cases(names)
    print(f"\n{len(names)} cases, {sum(4 + N_COND + len(MUTANTS) for _ in names)} oracle rounds: {time.time() - t0:.0f} s")
    return res


def _params():
    return [pytest.param(c, marks=[skip_m16] if c in SLOW else []) for c in CASES]


def _case(results, case):
    res = results[case]
    return res, dict(o64=res["o64"], o32s=res["o32s"], cond=res["cond"])


@pytest.mark.parametrize("case", _params())
def test_accepts_a_third_summation_order(results, case):
    """Correct fp32 arithmetic in an order the yardstick has not seen passes; its ratios calibrate what "1" means.
    On M16 it passes on every cooperative agent only: an adversary's nets fitted on its own data alone can leave the
    fp64 round by 1e-3 to 1e-2 of their norm in one fp32 order and not in another (module docstring), and which
    adversary does so depends on the order."""
    res, ref = _case(results, case)
    if case != "M16":
        R.yardstick(res["kernel"], msg=f"{case}: fp32 oracle, third order", **ref)
        return
    cfg = T16.loop_team("M16")
    _, flipped = R.yardstick_team(res["kernel"], labels=cfg["labels"], in_nodes=cfg["in_nodes"], max_flips=2,
                                  msg="M16: fp32 oracle, third order", **ref)
    assert all(cfg["labels"][i] == T16.M for i in flipped)


def _mutant_params():
    out = []
    for c in CASES:
        for m in MUTANTS:
            marks = [skip_m16] if c in SLOW else []
            if (c, m) in BLIND:
                marks.append(pytest.mark.xfail(strict=True, raises=AssertionError, reason=BLIND[c, m]))
            out.append(pytest.param(c, m, marks=marks))
    return out


@pytest.mark.parametrize("case,mutant", _mutant_params())
def test_rejects_wrong_arithmetic(results, case, mutant):
    """One input made subtly wrong: the yardstick must fail on a tensor the fault reaches (and, for the 1-ulp control,
    on none at all).  Prints the excess (ratio over the bound; above 1 fails) on those tensors and overall."""
    res, ref = _case(results, case)
    got, where = res[mutant]
    rows = R.yardstick_ratios(got, **ref)
    worst = max(rows, key=lambda row: row.excess)
    if where is None:                     # nothing may fail that the stand-in kernel without the mutant does not fail
        clean = {row.name: row.excess for row in R.yardstick_ratios(res["kernel"], **ref)}
        new = [row for row in rows if row.excess > 1 and not clean[row.name] > 1]
        print(f"\n{case} / {mutant} (control): largest excess {worst.excess:.2f} ({worst.name}), "
              f"{len(new)} tensors fail that passed without it")
        assert not new, f"the yardstick rejects a 1-ulp input change: {new[:3]}"
        return
    clean = {row.name: row.excess for row in R.yardstick_ratios(res["kernel"], **ref)}
    hit = max((row for row in rows if row.name.startswith(tuple(where)) and clean[row.name] <= 1),
              key=lambda row: row.excess)               # only tensors the stand-in passes on without the fault
    print(f"\n{case} / {mutant}: excess {hit.excess:.2f} on {hit.name} (where the fault acts); "
          f"largest anywhere {worst.excess:.2f} ({worst.name})")
    if (case, mutant) in WITHIN_NOISE:
        return
    assert hit.excess > 1, (f"{case} / {mutant}: the yardstick accepts the mutant on every tensor the fault reaches: "
                            f"{hit.name} is at {hit.excess:.2f} of its bound")


@pytest.mark.parametrize("case", _params())
def test_conditioning_term_changes_no_bound(results, case):
    """The fp64 round moves by no more than a few times the 2^-24 perturbation of its starting point, on every tensor
    of every case, M16's adversaries included: s_cond stays below max(s, floor ||o64||), so the conditioning term
    leaves every bound where the two fp32 samples put it.  M16's ten-epoch round is therefore not ill-conditioned to
    first order; what fp32 does there (test_accepts_a_third_summation_order) is not a matter of conditioning."""
    res, ref = _case(results, case)
    rows = R.yardstick_ratios(res["kernel"], **ref)
    worst = max(rows, key=lambda row: row.cond_rel)
    over = [row for row in rows if row.cond_rel > max(row.s_rel, R.YARD_FLOOR)]
    print(f"\n{case}: largest s_cond / ||o64|| = {worst.cond_rel:.1e} ({worst.name}), largest s / ||o64|| = "
          f"{max(row.s_rel for row in rows):.1e}; s_cond above max(s, floor) on {len(over)} tensors")
    assert worst.cond_rel <= COND_REL_MAX, worst
    assert not over, over[:3]


def test_n_cond_0_submits_the_three_rounds():
    """With n_cond = 0 yardstick_rounds runs exactly the fp64, fp32 and reassociated fp32 rounds, bit for bit what a
    direct call of the three gives (one epoch on 5 episodes of C2)."""
    r = build_round("c2", n_epochs=1, n_episodes=5)
    (res,) = R.yardstick_rounds([copy.deepcopy(r)], workers=1)
    assert len(res) == 3
    kw, n_act = r["kw"], 1
    alt_buf, alt_perms = R.reassociated(r["buf"], r["perms"], n_envs=1, n_actor_steps=kw["n_actor_steps"], n_act=n_act)
    direct = [R._oracle_round(copy.deepcopy(r["a64"]), r["labels"], r["in_nodes"], r["buf"], list(r["perms"]), kw),
              R._oracle_round(copy.deepcopy(r["a32"]), r["labels"], r["in_nodes"], r["buf"], list(r["perms"]), kw),
              R._oracle_round(copy.deepcopy(r["a32b"]), r["labels"], r["in_nodes"], alt_buf, alt_perms, kw)]
    for (ag, loss), (ag_d, loss_d) in zip(res, direct):
        a, b = R.round_tensors(ag), R.round_tensors(ag_d)
        assert a.keys() == b.keys()
        for name in a:
            assert a[name].dtype == b[name].dtype and np.array_equal(a[name], b[name]), name
        for key in loss:
            assert np.array_equal(loss[key], loss_d[key]), key
    (res4,) = R.yardstick_rounds([copy.deepcopy(r)], n_cond=2, workers=1)
    assert len(res4) == 5
    for name, x in R.round_tensors(res[0][0]).items():                       # the perturbed rounds are not the fp64 round
        assert np.array_equal(R.round_tensors(res4[0][0])[name], x)
    assert any(not np.array_equal(R.round_tensors(res4[3][0])[name], x) for name, x in R.round_tensors(res[0][0]).items())


def test_rotated_order_is_a_third_order():
    """reassociated(order="rotated") holds the same rows in every mini-batch as the other two orders, in an order that
    is neither of theirs, at N = 1 too."""
    r = build_round("c2", n_epochs=1, n_episodes=5)
    kw = dict(n_envs=1, n_actor_steps=r["kw"]["n_actor_steps"], n_act=1)
    (s0, *_), p0 = r["buf"], r["perms"]
    (s1, *_), p1 = R.reassociated(r["buf"], r["perms"], **kw)
    (s2, *_), p2 = R.reassociated(r["buf"], r["perms"], order="rotated", **kw)
    for a, b, c in zip(p0[:-1], p1[:-1], p2[:-1]):                           # the fit chains' (the last is the actor's)
        for k in range(0, len(a), 32):
            x, y, z = s0[a[k:k + 32]], s1[b[k:k + 32]], s2[c[k:k + 32]]
            assert np.array_equal(x, y[::-1]) and np.array_equal(x, np.roll(z, -(len(z) // 2), axis=0))
    assert not np.array_equal(s2, s0) and not np.array_equal(s2, s1)
