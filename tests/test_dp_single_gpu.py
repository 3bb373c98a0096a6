"""The data-parallel paths of the library on ONE GPU (the cross-rank peer-memory protocol itself needs two GPUs and is
tested by test_dp_gpu.py):
 (a) a bound world-1 exchange context at the C ABI: rcmarl_grad / rcmarl_team reduce through reduce_comm_kernel and
     rcmarl_minibatch_fit keeps its level-2 cells in the exchange buffer (its max_floats, its sequence numbers).  At
     world 1 the exchange adds nothing, so every result must be bitwise the unbound one.  Plus the context's refusals;
 (b) the same at Trainer level: a world-1 PeerComm bound under whole rollout + update rounds;
 (c) two ranks on one GPU over gloo without peer memory (the NCCL-fallback code path: rcmarl_grad -> all-reduce ->
     apply per step, the world scaling of every step coefficient, env_offset = rank * n_envs, the all-reduced episode
     means): injected rows against the fp64 oracle, and Philox rollouts against one process running all environments.
The exchange binding is process-global: every fixture that binds a context unbinds and destroys it when it ends."""
import ctypes as C
import datetime
import os
import sys
import traceback

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
import torch.multiprocessing as mp               # noqa: E402

from kernel_util import grad_ctas, load_kernels, rand_net, synth, to_dev   # noqa: E402
import team_util as T16                          # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
IN_S, IN_SA, IN_NS = 0, 1, 2                     # rcmarl_input_kind (include/rcmarl.h)
MSE, CE = 0, 1                                   # rcmarl_loss
MB = 32
NAN = float("nan")
SENTINEL = 7.25                                  # prefill of outputs a refused call must leave alone


@pytest.fixture(scope="module")
def K():
    return load_kernels()


# ==========================================================================================================
# (a) bound world-1 exchange context, C ABI level
# ==========================================================================================================
class Contexts:
    """World-1 exchange contexts made through the C ABI.  connect() maps no peer at world 1 (it skips its own rank), so
    no IPC handle is exported.  close() unbinds and destroys what is left."""

    def __init__(self, K):
        self.K, self.lib, self.live = K, K.L.lib(), []

    def create(self, max_floats):
        h = C.c_void_p()
        self.K.L.check(self.lib.rcmarl_comm_create(0, 1, max_floats, C.byref(h)), "rcmarl_comm_create")
        self.live.append(h)
        handles = C.create_string_buffer(self.lib.rcmarl_comm_handle_bytes())
        self.K.L.check(self.lib.rcmarl_comm_connect(h, handles), "rcmarl_comm_connect")
        return h

    def bind(self, h):
        self.K.L.check(self.lib.rcmarl_comm_bind(h), "rcmarl_comm_bind")

    def destroy(self, h):
        torch.cuda.synchronize()
        self.K.L.check(self.lib.rcmarl_comm_destroy(h), "rcmarl_comm_destroy")
        self.live = [x for x in self.live if x is not h]

    def close(self):
        torch.cuda.synchronize()
        self.lib.rcmarl_comm_bind(None)
        for h in self.live:
            self.lib.rcmarl_comm_destroy(h)
        self.live = []


@pytest.fixture
def contexts(K):
    c = Contexts(K)
    yield c
    c.close()


class Rows:
    """Seeded buffer rows of NA agents (B rows, grid nrow) on the device."""

    def __init__(self, K, rs, NA, B, nrow):
        s, ns, a, r = synth(rs, B, NA, nrow)
        self.NA, self.B = NA, B
        self.dsa, self.dns, self.dr = to_dev(K, np.concatenate([s, a], -1).reshape(B, -1), ns.reshape(B, -1), r[:, :, 0])

    def rows(self, K, time_idx=None, n_envs=1):
        if time_idx is None:
            return K.ops.make_rows(self.dsa, self.dns, self.dr, self.NA)
        return K.ops.make_rows(self.dsa, self.dns, self.dr, self.NA, 0, 0, time_idx, n_envs)


def d_in(NA, kind):
    return 3 * NA if kind == IN_SA else 2 * NA


class Scenario:
    """Host-side inputs of a fixed sequence of calls; run() executes it on fresh device copies (outputs prefilled with
    NaN) and returns every output.  The sequence interleaves the entry points that draw sequence numbers of a bound
    context: rcmarl_grad (MSE, 32 jobs at NA = 16), a persistent fit at the C2 width, rcmarl_grad (CE), rcmarl_team, a
    second persistent fit on the same cells, rcmarl_grad again."""

    def __init__(self, K, sms):
        rs = np.random.RandomState(2024)
        self.r16 = Rows(K, rs, 16, 3000, 10)
        kinds = ([IN_S, IN_SA, IN_NS] * 11)[:32]
        self.mse = []                                              # (net, kind, target or agent column, stride)
        for j, kind in enumerate(kinds):
            net = rand_net(rs, d_in(16, kind), 1)
            if j % 4 == 0:
                self.mse.append((net, kind, ("col", j % 16), 16))
            else:
                self.mse.append((net, kind, rs.randn(self.r16.B).astype(np.float32), 1))
        self.ce = [(rand_net(rs, 32, 5), i, rs.randn(self.r16.B).astype(np.float32)) for i in range(0, 16, 3)]
        # team jobs at NA = 16: messages of 16 agents per kind; job 1 has no sums, only agg_out
        self.msgs = {k: np.stack([K.nets.pack(rand_net(rs, d_in(16, k), 1)) for _ in range(16)]) for k in (IN_S, IN_SA)}
        self.team = [(IN_S, [0, 3, 5, 7, 9, 12], 2, True), (IN_SA, [1, 2, 4, 8, 10, 15], 1, False),
                     (IN_SA, [3, 4, 5, 6, 7, 8, 9, 10], 3, True), (IN_S, [15, 0, 1, 2], 1, True)]
        # persistent fits, NA = 5: the C2 width (4096 environments, 70 time rows: > 32 CTAs per chain) and a narrow one
        self.fits = []
        for N, T, E in ((4096, 70, 2), (64, 40, 3)):
            rows = Rows(K, rs, 5, N * T, 5)
            kinds5 = [IN_S, IN_SA, IN_S]
            nets = [rand_net(rs, d_in(5, k), 1) for k in kinds5]
            tgts = [rs.randn(N * T).astype(np.float32) for _ in kinds5]
            perms = np.stack([np.stack([rs.permutation(T) for _ in range(E)]) for _ in kinds5]).astype(np.int32)
            self.fits.append(dict(rows=rows, N=N, T=T, E=E, kinds=kinds5, nets=nets, tgts=tgts, perms=perms,
                                  lrs=[0.011, 0.013, 0.009]))
        wide = self.fits[0]
        assert min(grad_ctas(K, 5, wide["kinds"], MSE, MB * wide["N"], sms, balanced=True)) > 32

    def run(self, K):
        out = {}
        dev = K.dev
        ws = K.ops.workspace(K.L.MAX_JOBS, K.L.param_count(48, 1))
        cells = K.ops.MinibatchCells(K.L.MAX_JOBS, K.L.param_count(48, 1), dev)

        def grad_mse(tag):
            gj, sums = [], []
            for j, (net, kind, tgt, stride) in enumerate(self.mse):
                w = to_dev(K, K.nets.pack(net))[0]
                t = self.r16.dr[:, tgt[1]] if isinstance(tgt, tuple) else to_dev(K, tgt)[0]
                s = torch.full((w.numel() + 1,), NAN, device=dev)
                gj.append(K.ops.grad_job(w, t, s, kind, target_stride=stride))
                sums.append(s)
            K.ops.grad(self.r16.rows(K), gj, MSE, ws)
            out.update({f"{tag}/{j}": s for j, s in enumerate(sums)})

        def fit(k):
            f = self.fits[k]
            dperm = to_dev(K, f["perms"])[0]
            gj, aj, ws_ = [], [], []
            for c, (kind, net, tgt, lr) in enumerate(zip(f["kinds"], f["nets"], f["tgts"], f["lrs"])):
                w = to_dev(K, K.nets.pack(net))[0]
                s = torch.zeros(w.numel() + 1, device=dev)
                lo = torch.full((1,), NAN, device=dev)
                gj.append(K.ops.grad_job(w, to_dev(K, tgt)[0], s, kind, time_idx=dperm[c]))
                aj.append(K.ops.sgd_job(w, w, s, w.numel(), lr, loss_out=lo, loss_coef=1.0 / (f["N"] * f["T"])))
                ws_ += [w, lo]
            K.ops.minibatch_fit(f["rows"].rows(K, dperm, f["N"]), gj, aj, f["E"], f["T"], MB, 0.01, cells)
            out.update({f"fit{k}/{i}": t for i, t in enumerate(ws_)})

        grad_mse("mse0")
        fit(0)
        gj, sums = [], []
        for net, agent, delta in self.ce:
            w = to_dev(K, K.nets.pack(net))[0]
            s = torch.full((w.numel() + 1,), NAN, device=dev)
            gj.append(K.ops.grad_job(w, to_dev(K, delta)[0], s, IN_S, action_agent=agent))
            sums.append(s)
        K.ops.grad(self.r16.rows(K), gj, CE, ws)
        out.update({f"ce/{j}": s for j, s in enumerate(sums)})
        dmsgs = {k: to_dev(K, m)[0] for k, m in self.msgs.items()}
        tj = []
        for j, (kind, nodes, H, with_sums) in enumerate(self.team):
            s = torch.full((22,), NAN, device=dev) if with_sums else None
            agg = torch.full((self.r16.B,), NAN, device=dev)
            tj.append(K.ops.team_job(dmsgs[kind][nodes[0]], kind, dmsgs[kind], dmsgs[kind].shape[1], nodes, H, sums=s,
                                     agg_out=agg))
            out[f"team/agg{j}"] = agg
            if with_sums:
                out[f"team/sums{j}"] = s
        K.ops.team(self.r16.rows(K), tj, ws)
        fit(1)
        grad_mse("mse1")
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in out.items()}


def assert_equal_outputs(got, want, what):
    assert got.keys() == want.keys()
    for k in want:
        assert not torch.isnan(want[k]).any(), f"{what}: {k} not written"
        assert torch.equal(got[k], want[k]), f"{what}: {k} differs from the unbound call"


@pytest.fixture(scope="module")
def scenario(K):
    sc = Scenario(K, torch.cuda.get_device_properties(0).multi_processor_count)
    return sc, sc.run(K)                             # the unbound results, before any context exists


def test_bound_world1_context_matches_unbound_calls(K, contexts, scenario):
    """rcmarl_grad with 32 MSE jobs at NA = 16 (32 x 45 = 1 440 exchange items, more than the reduce grid: the item loop
    wraps), a CE launch, rcmarl_team with a job that has agg_out only, and two persistent fits on one cells buffer -- the
    first at the C2 width -- with rcmarl_grad / rcmarl_team between them: bitwise the unbound results, twice in a row on
    the same context (sequence numbers and slot parities keep moving across entry points)."""
    sc, want = scenario
    h = contexts.create(K.L.MAX_JOBS * 1536)
    contexts.bind(h)
    items = K.L.MAX_JOBS * -(-(K.L.param_count(48, 1) + 1) // 32)
    assert items > 2 * torch.cuda.get_device_properties(0).multi_processor_count
    for rep in range(2):
        assert_equal_outputs(sc.run(K), want, f"bound, pass {rep}")
    assert K.L.lib().rcmarl_comm_error(h) == 0


def test_comm_create_refusals(K):
    lib = K.L.lib()
    for rank, world, max_floats in ((0, 0, 1024), (0, 9, 1024), (1, 1, 1024), (2, 2, 1024), (-1, 1, 1024), (0, 1, 0),
                                    (0, 1, -5)):
        h = C.c_void_p()
        assert lib.rcmarl_comm_create(rank, world, max_floats, C.byref(h)) == -1, (rank, world, max_floats)
        assert h.value is None


def test_small_context_refuses_and_stays_usable(K, contexts):
    """A bound context with max_floats = 700 refuses rcmarl_grad (2 critic jobs: 2 x 662 floats), rcmarl_team (32 jobs:
    32 x 22) and rcmarl_minibatch_fit (3 chains) with RCMARL_ERR_ARG: sums, weights, loss slots and the whole cells
    buffer stay bitwise as they were.  Calls that fit then still give the unbound results, and after the context is
    destroyed the refused shapes run unbound again."""
    rs = np.random.RandomState(77)
    r5 = Rows(K, rs, 5, 640, 5)
    ws = K.ops.workspace(K.L.MAX_JOBS, K.L.param_count(48, 1))
    nets = [rand_net(rs, 10, 1) for _ in range(3)]
    tgt = to_dev(K, rs.randn(r5.B).astype(np.float32))[0]
    msgs = to_dev(K, np.stack([K.nets.pack(rand_net(rs, 10, 1)) for _ in range(5)]))[0]
    perms = np.stack([np.stack([rs.permutation(64) for _ in range(2)]) for _ in range(3)]).astype(np.int32)
    dperm = to_dev(K, perms)[0]
    n_c = K.L.param_count(10, 1)

    def grad(n_jobs):
        ws_ = [to_dev(K, K.nets.pack(nets[j]))[0] for j in range(n_jobs)]
        sums = torch.full((n_jobs, n_c + 1), SENTINEL, device=K.dev)
        return [K.ops.grad_job(ws_[j], tgt, sums[j], IN_S) for j in range(n_jobs)], sums

    def team(n_jobs):
        sums = torch.full((n_jobs, 22), SENTINEL, device=K.dev)
        jobs = [K.ops.team_job(msgs[j % 5], IN_S, msgs, n_c, [(j + k) % 5 for k in range(4)], 1, sums=sums[j])
                for j in range(n_jobs)]
        return jobs, sums

    def fit(n_chains, cells):
        w = torch.stack([to_dev(K, K.nets.pack(nets[c]))[0] for c in range(n_chains)])
        lo = torch.full((n_chains,), SENTINEL, device=K.dev)
        s = torch.zeros(n_chains, n_c + 1, device=K.dev)
        gj = [K.ops.grad_job(w[c], tgt, s[c], IN_S, time_idx=dperm[c]) for c in range(n_chains)]
        aj = [K.ops.sgd_job(w[c], w[c], s[c], n_c, 0.01, loss_out=lo[c:c + 1], loss_coef=1.0 / r5.B) for c in range(n_chains)]
        return (r5.rows(K, dperm, 10), gj, aj, 2, 64, MB, 0.01, cells), w, lo

    def unbound_results():
        out = []
        gj, sums = grad(1)
        K.ops.grad(r5.rows(K), gj, MSE, ws)
        tj, tsums = team(3)
        K.ops.team(r5.rows(K), tj, ws)
        args, w, lo = fit(1, K.ops.MinibatchCells(K.L.MAX_JOBS, K.L.param_count(48, 1), K.dev))
        K.ops.minibatch_fit(*args)
        torch.cuda.synchronize()
        out += [sums.cpu(), tsums.cpu(), w.cpu(), lo.cpu()]
        return out

    want = unbound_results()
    want_big = []
    gj, sums = grad(3)
    K.ops.grad(r5.rows(K), gj, MSE, ws)
    tj, tsums = team(32)
    K.ops.team(r5.rows(K), tj, ws)
    torch.cuda.synchronize()
    want_big += [sums.cpu(), tsums.cpu()]

    h = contexts.create(700)
    contexts.bind(h)
    gj, sums = grad(2)
    with pytest.raises(K.L.RcmarlError, match=r"rcmarl_grad: .*\(status -1,"):
        K.ops.grad(r5.rows(K), gj, MSE, ws)
    tj, tsums = team(32)
    with pytest.raises(K.L.RcmarlError, match=r"rcmarl_team: .*\(status -1,"):
        K.ops.team(r5.rows(K), tj, ws)
    cells = K.ops.MinibatchCells(K.L.MAX_JOBS, K.L.param_count(48, 1), K.dev)
    cells.buf.copy_(torch.randint(0, 256, cells.buf.shape, dtype=torch.uint8, device=K.dev))
    cells_before = cells.buf.clone()
    args, w, lo = fit(3, cells)
    w_before = w.clone()
    with pytest.raises(K.L.RcmarlError, match=r"rcmarl_minibatch_fit: .*\(status -1,"):
        K.ops.minibatch_fit(*args)
    torch.cuda.synchronize()
    assert bool((sums == SENTINEL).all()) and bool((tsums == SENTINEL).all())
    assert torch.equal(w, w_before) and bool((lo == SENTINEL).all())
    assert torch.equal(cells.buf, cells_before) and cells.seq == 1
    # the calls that fit the context are unaffected by the refusals before them
    got = unbound_results()
    for g, x in zip(got, want):
        assert torch.equal(g, x)
    assert K.L.lib().rcmarl_comm_error(h) == 0
    # destroying the bound context unbinds it: the shapes it refused run unbound
    contexts.destroy(h)
    gj, sums = grad(3)
    K.ops.grad(r5.rows(K), gj, MSE, ws)
    tj, tsums = team(32)
    K.ops.team(r5.rows(K), tj, ws)
    torch.cuda.synchronize()
    assert torch.equal(sums.cpu(), want_big[0]) and torch.equal(tsums.cpu(), want_big[1])


# ==========================================================================================================
# (b) bound world-1 exchange context, Trainer level
# ==========================================================================================================
def _team(name, rs):
    """Trainer keyword arguments of a tested team: c2 (the benchmark's 4 cooperative + 1 malicious agents, pretrained
    weights, 5x5 grid) or one of tests/team_util.TEAMS16 (16 agents, 10x10 grid, weights drawn from rs)."""
    if name == "c2":
        from golden_util import pretrained
        w, desired, labels = pretrained()
        return dict(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=[1] * 5,
                    fast_lr=[0.01] * 5)
    labels, in_nodes, w, desired, H, fast = T16.team16(name, rs)
    return dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, nrow=10, ncol=10, H=H, fast_lr=fast)


COMMON = dict(gamma=0.9, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100)


@pytest.fixture
def gloo_world1(tmp_path):
    """A world-1 gloo process group (PeerComm swaps its IPC handle through it) and the PeerComms made in it, closed
    (unbound, destroyed) before the group goes."""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'pg'}", rank=0, world_size=1,
                            timeout=datetime.timedelta(seconds=120))
    made = []
    yield made
    for c in made:
        c.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("team,N", [("c2", 64), ("M16", 8), ("X33", 8)])
def test_trainer_with_bound_world1_peer_comm_is_bitwise(K, gloo_world1, team, N):
    """Two rollout + update rounds with a bound world-1 PeerComm (the persistent fits' level-2 cells in the exchange
    buffer, every reduction through reduce_comm_kernel; X33 runs two fits per epoch) equal the same rounds without it:
    every parameter, Adam slot, loss and buffer row."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    kw = dict(_team(team, np.random.RandomState(11)), n_envs=N, seed=3, **COMMON)
    runs = []
    for bound in (False, True):
        tr = Trainer(**kw)
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        rounds = []
        for _ in range(2):
            rounds.append(tr.rollout_block())
            rounds.append(tr.update_round())
        torch.cuda.synchronize()
        runs.append((tr, rounds))
    (a, ra), (b, rb) = runs
    assert b.comm.bound and K.L.lib().rcmarl_comm_error(b.comm.handle) == 0
    for name in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v", "sa", "ns", "r"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert a.adam_t == b.adam_t
    for x, y in zip(ra, rb):
        if isinstance(x, dict):
            for k in x:
                np.testing.assert_array_equal(x[k], y[k], err_msg=k)
        else:
            np.testing.assert_array_equal(x[0], y[0]); np.testing.assert_array_equal(x[1], y[1])


# ==========================================================================================================
# (c) two ranks on one GPU over gloo, without peer memory
# ==========================================================================================================
# Seeds of the injected-rows cases: data on which the fp32 oracle itself stays within 1 % of the tolerance (with several
# adversaries among the neighbours, the clipped means make some data sets too ill-conditioned for fp32 arithmetic).
INJECTED = dict(N=8, T1=40, rounds=2, seeds=dict(c2=8, M16=17, X33=8))
PHILOX = dict(team="c2", N=64, seed=5)


def _shard(x, rank, world, N):
    """Rows of rank `rank`: its env columns [rank N / world, (rank + 1) N / world) of every time row (row = t N + e)."""
    h = N // world
    return x.reshape(-1, N, *x.shape[1:])[:, rank * h:(rank + 1) * h].reshape(-1, *x.shape[1:])


def _packed(tr):
    return torch.cat([tr.actor.flatten(), tr.critic.flatten(), tr.tr.flatten(), tr.critic_local.flatten(),
                      tr.adam_m.flatten(), tr.adam_v.flatten()]).cpu().numpy()


def _weights_flat(tr, n):
    return {f"w{i}_{m}_{k}": a for i in range(n) for m, net in enumerate(tr.get_weights(i)) for k, a in enumerate(net)}


def _run_case(case, rank, world):
    from rcmarl.trainer import Trainer
    out = {}
    if case["kind"] == "injected":
        N = case["N"]
        replay = T16.Replay()
        tr = Trainer(**case["team"], n_envs=N // world, rank=rank, world=world, perm_source=replay, **COMMON)
        assert tr.comm is None
        for k, (rows, perms) in enumerate(zip(case["rows"], case["perms"])):
            replay.load(perms)
            tr.load_rows(*[_shard(x, rank, world, N) for x in rows])
            for name, v in tr.update_round().items():
                out[f"r{k}_{name}"] = v
            assert replay.done()
    else:
        tr = Trainer(**case["team"], n_envs=case["N"] // world, rank=rank, world=world, seed=case["seed"], **COMMON)
        out["est"], out["ret"] = tr.rollout_block()
        B = tr.t_filled * tr.N
        out.update(sa=tr.sa[:B].cpu().numpy(), ns=tr.ns[:B].cpu().numpy(), r=tr.r[:B].cpu().numpy())
        tr.update_round()
    out["packed"] = _packed(tr)
    out.update(_weights_flat(tr, tr.n_real))
    return out


def _worker(rank, world, init_file, cases, out_dir):
    for p in (ROOT, os.path.join(ROOT, "resilient-consensus-based-marl_b200"), os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["RCMARL_PEER_COMM"] = "0"              # the all-reduce-per-step path; no peer-memory context
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=120))
    try:
        for name, case in cases.items():
            try:
                np.savez(os.path.join(out_dir, f"{name}.rank{rank}.npz"), **_run_case(case, rank, world))
            except Exception:                         # noqa: BLE001 -- reported by the parent's test of this case
                with open(os.path.join(out_dir, f"{name}.rank{rank}.err"), "w") as f:
                    f.write(traceback.format_exc())
        torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()


def _oracle_case(name):
    """Injected-rows case: data, the fp64 oracle's losses per round and final weights, the permutations it drew."""
    rs = np.random.RandomState(INJECTED["seeds"][name])
    team = _team(name, rs)
    labels, w = team["labels"], team["weights"]
    N, T1 = INJECTED["N"], INJECTED["T1"]
    agents = T16.oracle_agents(labels, w, team["H"], team["fast_lr"], COMMON["gamma"])
    oracle = T16.OracleRounds(agents, labels, team["in_nodes"], n_envs=N, n_epochs=COMMON["n_epochs"],
                              n_actor_steps=COMMON["max_ep_len"] * COMMON["n_ep_fixed"], buffer_size=COMMON["buffer_size"])
    rows, perms, losses = [], [], []
    for _ in range(INJECTED["rounds"]):
        data = T16.grid_rows(rs, T1 * N, len(labels), team["nrow"])
        loss, used = oracle.round(*data)
        rows.append(data)
        perms.append(used)
        losses.append(loss)
    case = dict(kind="injected", team=team, N=N, rows=rows, perms=perms)
    return case, losses, [ag.get_parameters() for ag in agents]


@pytest.fixture(scope="module")
def two_ranks(K, tmp_path_factory):
    """One 2-worker spawn that runs every case; -> (out_dir, oracle results by case, single-process Philox run)."""
    tmp = tmp_path_factory.mktemp("dp1")
    cases, oracle = {}, {}
    for name in ("c2", "M16", "X33"):
        case, losses, weights = _oracle_case(name)
        cases[name] = case
        oracle[name] = (losses, weights)
    cases["philox"] = dict(kind="philox", team=_team(PHILOX["team"], None), N=PHILOX["N"], seed=PHILOX["seed"])
    # the same Philox run in this process, all environments on one Trainer
    from rcmarl.trainer import Trainer
    tr = Trainer(**cases["philox"]["team"], n_envs=PHILOX["N"], seed=PHILOX["seed"], **COMMON)
    est, ret = tr.rollout_block()
    B = tr.t_filled * tr.N
    single = dict(est=est, ret=ret, sa=tr.sa[:B].cpu().numpy(), ns=tr.ns[:B].cpu().numpy(), r=tr.r[:B].cpu().numpy())
    tr.update_round()
    single["weights"] = [tr.get_weights(i) for i in range(tr.n_real)]
    del tr
    mp.spawn(_worker, args=(2, str(tmp / "pg"), cases, str(tmp)), nprocs=2, join=True)
    return tmp, oracle, single


def _load_ranks(out_dir, name):
    res = []
    for rank in range(2):
        err = out_dir / f"{name}.rank{rank}.err"
        if err.exists():
            pytest.fail(f"rank {rank} failed:\n{err.read_text()}")
        res.append(dict(np.load(out_dir / f"{name}.rank{rank}.npz")))
    return res


def _weights_of(res, n_nets):
    return [[[res[f"w{i}_{m}_{k}"] for k in range(6)] for m in range(n)] for i, n in enumerate(n_nets)]


@pytest.mark.parametrize("name", ["c2", "M16", "X33"])
def test_two_ranks_injected_rows_match_oracle(two_ranks, name):
    """2 ranks x 4 environments over gloo (rcmarl_grad -> all-reduce -> apply per step, the adversaries' chains in
    groups of at most 32 for X33) against the oracle's update rounds over all 8 environments in fp64; the ranks'
    parameters and Adam slots are bitwise equal (each chunk is reduced once)."""
    out_dir, oracle, _ = two_ranks
    r0, r1 = _load_ranks(out_dir, name)
    assert np.array_equal(r0["packed"], r1["packed"]), "replicated parameters diverged between ranks"
    losses, want_w = oracle[name]
    for k, want in enumerate(losses):
        for key in ("critic_loss", "TR_loss", "actor_loss"):
            for rank, res in enumerate((r0, r1)):
                np.testing.assert_allclose(res[f"r{k}_{key}"], want[key], rtol=2e-3, atol=2e-5,
                                           err_msg=f"round {k} {key} rank {rank}")
    got = _weights_of(r0, [len(w) for w in want_w])
    for i, want in enumerate(want_w):
        T16.close_w(got[i], want, msg=f"agent {i}")


def test_two_ranks_philox_rollout_match_one_process(two_ranks):
    """C2 at 64 environments as 2 ranks x 32: each rank's buffer rows are bitwise its env columns of the one-process run
    (env_offset = rank x 32 keys the Philox streams), the all-reduced episode means match, and after one update round
    the weights match as in test_dp_gpu.py."""
    out_dir, _, single = two_ranks
    ranks = _load_ranks(out_dir, "philox")
    assert np.array_equal(ranks[0]["packed"], ranks[1]["packed"]), "replicated parameters diverged between ranks"
    N = PHILOX["N"]
    for rank, res in enumerate(ranks):
        for key in ("sa", "ns", "r"):
            assert np.array_equal(res[key], _shard(single[key], rank, 2, N)), f"{key} rows of rank {rank}"
        for key in ("est", "ret"):
            np.testing.assert_allclose(res[key], single[key], rtol=1e-6, atol=1e-7, err_msg=f"{key} rank {rank}")
    got = _weights_of(ranks[0], [len(w) for w in single["weights"]])
    for i, want in enumerate(single["weights"]):
        T16.close_w(got[i], want, rtol=2e-3, atol=2e-5, msg=f"agent {i}")
