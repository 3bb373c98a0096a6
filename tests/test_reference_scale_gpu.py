"""Update rounds at the reference hyper-parameters (bench.HYPER = main.py's defaults: n_epochs = 10, buffer_size = 2000,
blocks of 50 episodes x 20 steps) against the fp64 oracle, in the regime bench.py times: a buffer of 3000 time rows of
which the round trims 1000, 94 mini-batches per epoch (the last of 24 time rows) in the adversaries' fits, an actor
window of 1000 rows starting at row 2000 x N, 5 Adam mini-batches of 200 time rows, and Keras-Adam step counts that
carry across rounds.

Each round is teacher-forced as test_rollout_philox_gpu.py (d) does: before every block the oracle agents are loaded
from the Trainer; the block's rows are compared exactly (tie episodes excluded) and its logged means at the forward
tolerances; the update round runs on the Trainer's buffer with the Trainer's own shuffles (default_perm_source); the
kept buffer must be the newest buffer_size time rows.  Weights and Adam m and v are held to the fp32-spread yardstick
of rollout_oracle.yardstick: within c = 8 times (12 in the max norm) the larger of the spread s of two fp32 oracle
rounds (two summation orders) around the fp64 round, and 1e-6 of the tensor's norm.  The oracle rounds use the
kernel's fp32 Adam constants (O.KerasAdam with fp32_betas, rollout_oracle.with_kernel_adam).  Adam step counts are compared exactly, losses at the
whole-round tolerance.

Measured on an H100 80GB HBM3, largest ||gpu - o64|| / s per round (normwise; max norm in brackets):
  bench schedule N = 1, T = 3000 x 3:                 1.3 (1.4), 5.5 (7.1), 1.1 (1.1)
  main.py schedule N = 1, T = 1000 / 2000 / 3000:     1.8 (2.4), 1.4 (1.8), 3.2 (4.4)
  bench schedule N = 64, T = 3000:                    3.6 (3.6)
  Greedy + Faulty N = 4, T = 1000 / 2000:             1.1 (1.1), 5.3 (6.1)
  fit at N = 256 (persistent kernel, step loop):      1.0 (1.0), 1.0 (1.1)
  fit at N = 4096, persistent kernel vs step loop:    0.23 of the N = 256 relative spread
M16 (N = 2, main.py's schedule) is judged by rollout_oracle.yardstick_team, which excuses per round a bounded number of
adversaries whose fp32 mini-batch fits met a leaky-ReLU sign flip, with the cooperative agents that hear them.  Measured
on the same card (700 W power limit, `pytest -m gpu tests/test_reference_scale_gpu.py -q -s`), tensors within the plain
bound, and the largest ratio over the agents without a miss:
  M16 ten epochs, T = 1000 / 2000:                    472 of 504 (6.9; agents 3, 13 -> 10), 503 of 504 (4.6; agent 9)
  M16 one epoch,  T = 1000 / 2000:                    486 of 504 (1.4; agent 13 -> 8, 10, 12), 504 of 504 (1.5)
The median over tensors of ||o32 - o32b|| / s is 0.3 to 0.9 in six of the nine rounds, so there s measures rounding.
It is much smaller in three: 0.12 in bench N = 1 round 2, 0.14 in the N = 256 fit and 0.06 in Greedy + Faulty round 0.
There the two fp32 orders agree with each other far better than with fp64, so s there is mostly a systematic fp32 /
fp64 difference rather than the rounding spread, and the bound is that much looser.  The file takes about 5
minutes, most of it the N = 64 oracle round.

test_fit_at_benchmark_width runs the Malicious agent's three mini-batch chains (10 epochs x 94 steps) on a Trainer's
real buffer: at N = 256 against the oracle's fit_minibatch by the same yardstick, and at the benchmark's N = 4096,
where the oracle is too slow, the persistent kernel against the per-step rcmarl_grad -> rcmarl_sgd_apply loop.

Each test prints, per round, the largest ||gpu - o64|| / max(s, floor) over all tensors and the median over tensors
of ||o32 - o32b|| / s (about 1: s measures rounding; much less: a systematic fp32 / fp64 difference).
Most of the wall time is the CPU oracle, which runs in parallel worker processes."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import bench                                          # noqa: E402  (workload / HYPER only: importing it runs nothing)
import rollout_oracle as R                            # noqa: E402
import team_util as T16                               # noqa: E402
from kernel_util import close, load_kernels, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                 # noqa: E402  (checker only)

f32, f64 = np.float32, np.float64
SEED = 1234                                           # bench.py's
HYPER = bench.HYPER


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def teacher_forced_rounds(cfg, schedule, n_updates, seed=SEED):
    """A Trainer on cfg (bench.workload or a loop_team with HYPER).  schedule "bench": two blocks without an update,
    then n_updates x (block + update_round), as bench.py's steady state; "main": block + update_round from the start,
    as train_RPBCAC.  Checks every block's rows and means and every kept buffer; returns what the update rounds need
    for the yardstick, with the Trainer's results."""
    from rcmarl.trainer import Trainer
    tr = Trainer(**cfg, seed=seed)
    n, N = len(cfg["labels"]), cfg["n_envs"]
    L_, ne = cfg["max_ep_len"], cfg["n_ep_fixed"]
    block = L_ * ne
    perms = R.default_perm_source(seed)
    rounds = []
    n_blocks = n_updates + (2 if schedule == "bench" else 0)
    for k in range(n_blocks):
        agents = R.oracle_agents_from_trainer(tr)
        draws = R.rollout_draws(seed, env_offset=0, n_envs=N, episode_offset=k * ne, n_episodes=ne, max_ep_len=L_,
                                n_slots=tr.NA, n_active=n, nrow=cfg["nrow"], ncol=cfg["ncol"])
        t0 = tr.t_filled
        est_m, ret_m = tr.rollout_block()
        want, est, ret = R.oracle_rollout(agents, cfg["desired"], cfg["nrow"], cfg["ncol"], draws, cfg["gamma"])
        ok = R.check_rows(R.trainer_rows(tr, t0, t0 + block), want, ne, L_, N)
        close(est_m, est.mean(1), rtol=1e-5, atol=3e-6, err_msg=f"block {k} est")
        full = ok.all(1)
        close(ret_m[full], ret[full].mean(1), rtol=1e-5, atol=1e-5, err_msg=f"block {k} ret")
        if schedule == "bench" and k < 2:
            continue
        T = tr.t_filled
        buf = R.trainer_rows(tr, 0, T)
        kw = dict(n_envs=N, n_epochs=cfg["n_epochs"], n_actor_steps=block, common_reward=cfg.get("common_reward", False))
        r = dict(T=T, labels=cfg["labels"], in_nodes=cfg["in_nodes"], buf=buf, kw=kw, a64=R.with_kernel_adam(agents),
                 a32=R.with_kernel_adam(R.oracle_agents_from_trainer(tr, f32)),
                 a32b=R.with_kernel_adam(R.oracle_agents_from_trainer(tr, f32)),
                 perms=R.round_perms(perms, cfg["labels"], T, n_epochs=cfg["n_epochs"], n_actor_steps=block))
        r["loss"] = tr.update_round()
        got = R.oracle_agents_from_trainer(tr)
        r["got"], r["got_t"] = R.round_tensors(got), [ag.adam.t for ag in got]
        keep = min(T, cfg["buffer_size"])
        assert tr.t_filled == keep
        for g, x in zip(R.trainer_rows(tr, 0, keep), buf):
            assert np.array_equal(g, x[-keep * N:]), f"block {k}: kept buffer"
        rounds.append(r)
    return rounds


def check_rounds(rounds, case, max_flips=None, losses=True):
    """The three oracle rounds per update round (in parallel) and the yardstick; prints the ratios per round.
    max_flips: judge by rollout_oracle.yardstick_team, which excuses that many adversaries per round whose fits met a
    leaky-ReLU sign flip (and the cooperative agents that hear them).  losses=False: after ten epochs a flipped fit's
    logged loss is off by as much as its net (measured: up to 15 times the whole-round tolerance), so M16's ten-epoch
    rounds compare tensors only."""
    results = R.yardstick_rounds(rounds)
    for k, (r, res) in enumerate(zip(rounds, results)):
        (a64, l64), (a32, l32), (a32b, l32b) = res
        assert r["got_t"] == [ag.adam.t for ag in a64], f"{case} round {k}: Adam step counts"
        ref = (r["got"], R.round_tensors(a64), [R.round_tensors(a32), R.round_tensors(a32b)])
        msg = f"{case} round {k} (T = {r['T']})"
        if max_flips is None:
            R.yardstick(*ref, msg=msg)
        else:
            R.yardstick_team(*ref, labels=r["labels"], in_nodes=r["in_nodes"], max_flips=max_flips, msg=msg)
        for key in ("critic_loss", "TR_loss", "actor_loss") if losses else ():
            np.testing.assert_allclose(r["loss"][key], l64[key], rtol=2e-3, atol=2e-5, err_msg=f"{case} round {k} {key}")
    return results


def test_bench_schedule_n1(K):
    """bench.py's schedule at N = 1: two blocks without an update, then three steps of block + update_round, each at
    T = 3000 with a trim of 1000 rows; Adam t = 1, 2, 3 for the cooperative agents, 5, 10, 15 for the Malicious one."""
    cfg = bench.workload("C2", 1)
    rounds = teacher_forced_rounds(cfg, "bench", 3)
    assert [r["T"] for r in rounds] == [3000] * 3
    check_rounds(rounds, "bench N=1")
    mal = cfg["labels"].index("Malicious")
    assert [r["got_t"][0] for r in rounds] == [1, 2, 3]
    assert [r["got_t"][mal] for r in rounds] == [5, 10, 15]


def test_main_schedule_n1(K):
    """main.py's schedule (train_RPBCAC) at N = 1: an update after every block, T = 1000, 2000, 3000 (the first
    trim)."""
    rounds = teacher_forced_rounds(bench.workload("C2", 1), "main", 3)
    assert [r["T"] for r in rounds] == [1000, 2000, 3000]
    check_rounds(rounds, "main N=1")


def test_bench_schedule_n64(K):
    """bench.py's schedule at N = 64, one step (the oracle round takes minutes): the gathered mini-batch rows take
    grad_kernel's bulk-copy (TMA) staging branch."""
    rounds = teacher_forced_rounds(bench.workload("C2", 64), "bench", 1)
    assert rounds[0]["T"] == 3000
    check_rounds(rounds, "bench N=64")


@pytest.mark.parametrize("name,N,n_updates", [("greedy_faulty", 4, 2), ("M16", 2, 2)])
def test_other_teams_main_schedule(K, name, N, n_updates):
    """Greedy + Faulty with common_reward, and the 16-agent M16 team (16 mini-batch chains, per-agent H and fast_lr), at
    the reference hyper-parameters on main.py's schedule.  M16 is judged by yardstick_team: measured, Greedy agent 3 and
    Malicious agent 13 (with cooperative agent 10, which hears 13) leave the bound at T = 1000 and one Adam slot of
    Malicious agent 9 at T = 2000; the other 472 and 503 of 504 tensors are held."""
    cfg = {**HYPER, **T16.loop_team(name), "n_envs": N}
    rounds = teacher_forced_rounds(cfg, "main", n_updates)
    check_rounds(rounds, f"{name} N={N}", max_flips=2 if name == "M16" else None, losses=name != "M16")


def test_m16_reference_buffer_single_epoch(K):
    """M16 on the same grid, N = 2, buffer (T = 1000, 2000) and block sizes, with n_epochs = 1: the launches of the
    ten-epoch round (16 chains, 32 and 63 mini-batches per inner epoch, the actor window, per-agent H and fast_lr)
    without ten epochs in which sign flips compound.  Measured: at T = 2000 all 504 tensors pass the plain yardstick
    (largest ratio 1.45); at T = 1000 Malicious agent 13's critic meets a flip (1.3e-4 of its norm) that cooperative
    agents 8, 10 and 12 hear (2.4e-4 on agent 8's critic), and the other 486 tensors pass (1.37).  So one flip is
    excused per round."""
    cfg = {**HYPER, **T16.loop_team("M16"), "n_envs": 2, "n_epochs": 1}
    rounds = teacher_forced_rounds(cfg, "main", 2)
    assert [r["T"] for r in rounds] == [1000, 2000]
    check_rounds(rounds, "M16 N=2, one epoch", max_flips=1)


# --------------------------------------------------------------------------------------------- the benchmark's width
def _forward64(w, x):
    """The fp64 value of a net (six Keras arrays) on device rows x."""
    W1, b1, W2, b2, W3, b3 = (torch.as_tensor(np.asarray(a, f64), device=x.device) for a in w)
    lrelu = torch.nn.functional.leaky_relu
    return (lrelu(lrelu(x @ W1 + b1, 0.1) @ W2 + b2, 0.1) @ W3 + b3)[:, 0]


def _malicious_chains(K, tr, i, N, T, host=True):
    """The three chains Trainer._minibatch_sgd fits for Malicious agent i, on the first N environments of its buffer:
    [(weights, input kind, fp32 target on the device)] for critic_local on r_i + gamma V_local(ns), TR on -r_coop and
    critic on -r_coop + gamma V(ns) (targets formed in fp64 and rounded once: the fit is what is under test), the
    device rows (sa, ns, r) and, if host, the fp64 host inputs per kind for the oracle (else None)."""
    NA, n = tr.NA, tr.n_real
    sa, ns, r = (x[:T * tr.N].view(T, tr.N, -1)[:, :N].reshape(T * N, -1).contiguous() for x in (tr.sa, tr.ns, tr.r))
    x_ns = ns.view(-1, NA, 2)[:, :n].reshape(T * N, -1).double()
    ag = R.oracle_agents_from_trainer(tr)[i]
    coop = [j for j in range(n) if tr.labels[j] == "Cooperative"]
    neg_r_coop = -r[:, coop].double().sum(1) / len(coop)
    chains = [(ag.critic_local_weights, K.L.IN_S, r[:, i].double() + tr.gamma * _forward64(ag.critic_local_weights, x_ns)),
              (ag.TR, K.L.IN_SA, neg_r_coop),
              (ag.critic, K.L.IN_S, neg_r_coop + tr.gamma * _forward64(ag.critic, x_ns))]
    if host:
        x = sa.view(-1, NA, 3)[:, :n]
        host = {K.L.IN_S: x[..., :2].reshape(T * N, -1).double().cpu().numpy(),
                K.L.IN_SA: x.reshape(T * N, -1).double().cpu().numpy()}
    return [(w, kind, tgt.float().contiguous()) for w, kind, tgt in chains], (sa, ns, r), host or None


def _gpu_fit(K, tr, chains, rows_dev, dperm, N, T, lr, persistent):
    """The chains' fit through ops.minibatch_fit (the persistent kernel) or ops.minibatch_steps (per step
    rcmarl_grad -> rcmarl_sgd_apply) -> name -> array, as _fit_tensors."""
    ws, losses, gj, aj = [], [], [], []
    for c, (w, kind, tgt) in enumerate(chains):
        wd = to_dev(K, K.nets.pack(w))[0]
        sums = torch.zeros(wd.numel() + 1, device=K.dev)
        lo = torch.zeros(1, device=K.dev)
        gj.append(K.ops.grad_job(wd, tgt, sums, kind, time_idx=dperm[c]))
        aj.append(K.ops.sgd_job(wd, wd, sums, wd.numel(), lr, loss_out=lo, loss_coef=1.0 / (T * N)))
        ws.append(wd)
        losses.append(lo)
    rows = K.ops.make_rows(*rows_dev, tr.NA, 0, 0, dperm, N)
    E, MB = tr.mb_epochs, tr.mb_times
    if persistent:
        K.ops.minibatch_fit(rows, gj, aj, E, T, MB, lr, K.ops.MinibatchCells())
    else:
        K.ops.minibatch_steps(rows, gj, aj, E, T, MB, [lr] * len(chains))
    torch.cuda.synchronize()
    return _fit_tensors([K.nets.unpack(w.cpu().numpy(), len(chains[c][0][0]), 1) for c, w in enumerate(ws)],
                        [lo.item() for lo in losses])


def _fit_tensors(nets, losses):
    out = {}
    for c, (w, loss) in enumerate(zip(nets, losses)):
        for k, x in enumerate(w):
            out[f"chain {c} array {k}"] = x
        out[f"chain {c} loss"] = np.float64(loss)
    return out


def test_fit_at_benchmark_width(K):
    """The Malicious agent's three mini-batch chains (critic_local, TR, critic; E = 10, mb_times = 32, 94 steps per
    epoch, the last of 24 time rows) on a Trainer's real buffer after bench.py's two blocks plus one (T = 3000):
    at N = 256 the persistent kernel and the step loop against O.fit_minibatch by the yardstick (three oracle fits per
    chain: fp64, fp32, fp32 reassociated); at N = 4096, 2 820 steps over 131 072 rows per mini-batch, the persistent
    kernel against the step loop, normwise within c times the relative fp32 spread measured at N = 256 (or the floor)."""
    from rcmarl.trainer import Trainer
    cfg = bench.workload("C2", 4096)
    tr = Trainer(**cfg, seed=SEED)
    for _ in range(3):
        tr.rollout_block()
    T = tr.t_filled
    assert T == 3000
    i = cfg["labels"].index("Malicious")
    E, MB, lr = tr.mb_epochs, tr.mb_times, tr.fast_lr[i]
    assert (E, MB, -(-T // MB), T % MB) == (10, 32, 94, 24)
    rs = np.random.RandomState(3)
    perms = np.stack([np.stack([rs.permutation(T) for _ in range(E)]) for _ in range(3)]).astype(np.int32)   # [C,E,T]
    dperm = to_dev(K, perms)[0]

    # N = 256 against the oracle
    N = 256
    chains, rows_dev, host = _malicious_chains(K, tr, i, N, T)
    got = {p: _gpu_fit(K, tr, chains, rows_dev, dperm, N, T, lr, p) for p in (True, False)}
    jobs = []
    for c, (w, kind, tgt) in enumerate(chains):
        x, y = host[kind], tgt.double().cpu().numpy().reshape(-1, 1)
        (xb, yb), pb = R.reassociated((x, y), list(perms[c]), n_envs=N, n_actor_steps=T, n_act=0, mb_times=MB)
        for dt, (xx, yy, pp) in ((f64, (x, y, perms[c])), (f32, (x, y, perms[c])), (f32, (xb, yb, pb))):
            jobs.append((O.cast_weights(w, dt), xx.astype(dt), yy.astype(dt), lr, E, MB * N,
                         [O.expand_time_perm(p, N) for p in pp]))
    res = R.parallel_map(O.fit_minibatch, jobs)
    o = [_fit_tensors([res[3 * c + v][0] for c in range(3)], [res[3 * c + v][1] for c in range(3)]) for v in range(3)]
    s_rel = {name: max(np.linalg.norm(np.asarray(oo[name], f64) - x) for oo in o[1:]) / np.linalg.norm(x)
             for name, x in o[0].items()}
    for p in (True, False):
        R.yardstick(got[p], o[0], o[1:], msg=f"fit N={N} {'persistent kernel' if p else 'step loop'}")
        for c in range(3):
            np.testing.assert_allclose(got[p][f"chain {c} loss"], o[0][f"chain {c} loss"], rtol=1e-4)

    # N = 4096: the persistent kernel against the step loop
    N = tr.N
    chains, rows_dev, _ = _malicious_chains(K, tr, i, N, T, host=False)
    fit, loop = (_gpu_fit(K, tr, chains, rows_dev, dperm, N, T, lr, p) for p in (True, False))
    worst = 0.0
    for name, x in loop.items():
        x = np.asarray(x, f64)
        tol = max(s_rel[name], R.YARD_FLOOR) * np.linalg.norm(x)
        err = np.linalg.norm(np.asarray(fit[name], f64) - x)
        assert err <= R.YARD_C * tol, f"N={N} {name}: ||persistent - step loop|| = {err:.3e} > {R.YARD_C} x {tol:.3e}"
        worst = max(worst, err / tol)
    print(f"\nfit N={N} persistent vs step loop: ||diff|| / (N=256 relative spread x ||loop||) = {worst:.2f}")
