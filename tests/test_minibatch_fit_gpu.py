"""rcmarl_minibatch_fit (csrc/minibatch_persist.cuh) against the fp64 oracle's fit_minibatch, with the chain mixes the
trainer launches and across calls that share one cells buffer:
 - the chains Trainer builds for [Cooperative, Malicious, Greedy, Cooperative, Malicious] in one launch: critic_local
   chains without loss_out, the Greedy team-reward target as the column view r[:, i] (target_stride = NA), a learning
   rate per chain (coef = 0 takes the call's lr), loss_out overwritten (loss_accumulate = 0) or added to (= 1);
 - RCMARL_MAX_JOBS chains of mixed kinds, and one more refused;
 - three fits in a row on one MinibatchCells with different CTA grids, each checked against the oracle;
 - the 32-bit sequence-number limits: ops restarting on clean cells, the largest accepted seq_first, refused values;
 - the argument checks of the C ABI: every refusal leaves the weights and the whole cells buffer bitwise unchanged.
The permutations are injected (oracle: O.expand_time_perm of the same time-row tables).  The second reference is the
per-step loop ops.minibatch_steps (rcmarl_grad -> rcmarl_sgd_apply) at world 1.

Tolerances as in test_kernels_gpu.py: fits of a few steps rtol 2e-4 / atol 2e-6 against the oracle and 1e-5 / 1e-6
against the step loop; fits of E = 10 epochs the whole-round tolerance rtol 1e-3 / atol 5e-5 (DESIGN.md section 2);
epoch-0 losses rtol 1e-4."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from kernel_util import grad_ctas, load_kernels, rand_net, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
IN_S, IN_SA, IN_NS = 0, 1, 2          # rcmarl_input_kind (include/rcmarl.h)
MSE = 0                               # rcmarl_loss
OK, ERR_ARG, ERR_WORKSPACE = 0, -1, -2
NA = 5
MB = 32                               # mini-batch: 32 time rows x n_envs environments (Appendix C)
SEQ_LIMIT = 0xFFFFFFFF                # seq_first + steps must stay below it
MIXED = ['Cooperative', 'Malicious', 'Greedy', 'Cooperative', 'Malicious']
SHORT = dict(rtol=2e-4, atol=2e-6)    # weights vs the oracle, fits of up to ~9 steps
SHORT_LOOP = dict(rtol=1e-5, atol=1e-6)
ROUND = dict(rtol=1e-3, atol=5e-5)    # E = 10 epochs (the trainer's mb_epochs)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


@pytest.fixture(scope="module")
def SMS(K):
    return torch.cuda.get_device_properties(0).multi_processor_count


def d_in(kind):
    return 3 * NA if kind == IN_SA else 2 * NA


class Buf:
    """Seeded buffer rows of T time rows x N environments (row = t * N + e), on the host (flattened per input kind) and
    the device.  room_for_16: the device arrays sit at the start of allocations wide enough for 16 agents."""

    def __init__(self, K, rs, N, T, room_for_16=False):
        B = N * T
        s, ns, a, r = synth(rs, B, NA, 5)
        self.N, self.T, self.B = N, T, B
        self.x = {IN_S: s.reshape(B, -1), IN_SA: np.concatenate([s, a], -1).reshape(B, -1), IN_NS: ns.reshape(B, -1)}
        self.r = r[:, :, 0]
        dev = to_dev(K, self.x[IN_SA], self.x[IN_NS], self.r)
        if room_for_16:
            dev = [_padded(K, d, 16 // NA + 1) for d in dev]
        self.dsa, self.dns, self.dr = dev

    def rows(self, K, dperm):
        return K.ops.make_rows(self.dsa, self.dns, self.dr, NA, 0, 0, dperm, self.N)


def _padded(K, t, factor):
    """t copied to the start of a zeroed allocation factor times its size (a view of the same shape)."""
    big = torch.zeros(t.numel() * factor, device=K.dev)
    big[:t.numel()].copy_(t.reshape(-1))
    return big[:t.numel()].view(t.shape)


class Chain:
    """One mini-batch chain: net, input kind, target (host array and device tensor / column view), per-chain learning
    rate coef (0: the call's lr) and loss slot: loss None (no loss_out), or loss_out prefilled with loss_init and either
    overwritten (acc = 0) or added to (acc = 1)."""

    def __init__(self, rs, kind, tgt, dtgt, stride=1, coef=0.0, loss=True, acc=1, loss_init=0.0):
        self.kind, self.tgt, self.dtgt, self.stride, self.coef = kind, tgt, dtgt, stride, coef
        self.net = rand_net(rs, d_in(kind), 1)
        self.loss, self.acc, self.loss_init = loss, acc, loss_init

    def lr(self, call_lr):
        return self.coef if self.coef > 0 else call_lr


def random_target(K, rs, buf):
    t = rs.randn(buf.B).astype(np.float32)
    return t, to_dev(K, t)[0]


def trainer_chains(K, rs, buf, labels):
    """The chains Trainer._minibatch_sgd builds for `labels` (rcmarl/trainer.py, node order): per Malicious agent its
    critic_local fit (no loss_out), its team-reward fit on -r_coop and its critic fit; per Greedy agent its team-reward
    fit on its own reward column r[:, i] (target_stride = NA) and its critic fit.  The critics' TD targets are random
    here.  Learning rates differ per chain and one chain has coef = 0; loss slots alternate between overwritten
    (prefilled with garbage) and added to (prefilled with a known value)."""
    coop = [i for i, lab in enumerate(labels) if lab == 'Cooperative']
    neg_r_coop = (-(buf.r[:, coop].astype(f64).sum(1) / len(coop))).astype(np.float32)
    d_neg = to_dev(K, neg_r_coop)[0]
    chains = []
    for i, lab in enumerate(labels):
        if lab == 'Malicious':
            chains.append(Chain(rs, IN_S, *random_target(K, rs, buf), loss=False))
            chains.append(Chain(rs, IN_SA, neg_r_coop, d_neg))
            chains.append(Chain(rs, IN_S, *random_target(K, rs, buf)))
        elif lab == 'Greedy':
            chains.append(Chain(rs, IN_SA, buf.r[:, i].copy(), buf.dr[:, i], stride=NA))
            chains.append(Chain(rs, IN_S, *random_target(K, rs, buf)))
    coefs = [0.010, 0.013, 0.0, 0.008, 0.016, 0.011, 0.007, 0.014]
    k = 0
    for ch, coef in zip(chains, coefs * (len(chains) // len(coefs) + 1)):
        ch.coef = coef
        if ch.loss:
            ch.acc = k % 2
            ch.loss_init = 0.25 if ch.acc else 777.0
            k += 1
    return chains


def perm_tables(K, rs, n_chains, E, T):
    p = np.stack([np.stack([rs.permutation(T) for _ in range(E)]) for _ in range(n_chains)]).astype(np.int32)  # [C, E, T]
    return p, to_dev(K, p)[0]


def jobs(K, buf, chains, dperm, room_for_16=False):
    """Weights (fresh copies of the chains' nets), loss slots and the grad / sgd job lists of one fit."""
    ws, losses, gj, aj = [], [], [], []
    for c, ch in enumerate(chains):
        w = to_dev(K, K.nets.pack(ch.net))[0]
        if room_for_16:
            w = _padded(K, w, K.L.param_count(48, 1) // w.numel() + 1)
        n = w.numel()
        sums = torch.zeros(n + 1, device=K.dev)
        lo = torch.full((1,), ch.loss_init, device=K.dev) if ch.loss else None
        gj.append(K.ops.grad_job(w, ch.dtgt, sums, ch.kind, target_stride=ch.stride, time_idx=dperm[c]))
        aj.append(K.ops.sgd_job(w, w, sums, n, ch.coef, loss_out=lo, loss_coef=1.0 / buf.B, loss_accumulate=ch.acc))
        ws.append(w)
        losses.append(lo)
    return ws, losses, gj, aj


def fetch(ws, losses):
    torch.cuda.synchronize()
    return [w.cpu().numpy() for w in ws], [None if lo is None else float(lo.item()) for lo in losses]


def run_persistent(K, buf, chains, dperm, E, lr, cells):
    ws, losses, gj, aj = jobs(K, buf, chains, dperm)
    K.ops.minibatch_fit(buf.rows(K, dperm), gj, aj, E, buf.T, MB, lr, cells)
    return fetch(ws, losses)


def run_steps(K, buf, chains, dperm, E, lr):
    ws, losses, gj, aj = jobs(K, buf, chains, dperm)
    K.ops.minibatch_steps(buf.rows(K, dperm), gj, aj, E, buf.T, MB, [ch.lr(lr) for ch in chains])
    return fetch(ws, losses)


def check_against_oracle(K, buf, chains, perms, E, lr, got, tol, loop=None, loop_tol=None):
    """Every chain's weights and loss slot against fit_minibatch in fp64 with that chain's own learning rate, target and
    permutations (and against the step loop's result `loop`)."""
    w_got, l_got = got
    for c, ch in enumerate(chains):
        w64, l64 = O.fit_minibatch(O.cast_weights(ch.net, f64), buf.x[ch.kind].astype(f64),
                                   ch.tgt.astype(f64).reshape(-1, 1), ch.lr(lr), E, MB * buf.N,
                                   [O.expand_time_perm(perms[c, e], buf.N) for e in range(E)])
        msg = f"chain {c} (kind {ch.kind}, stride {ch.stride}, lr {ch.lr(lr)})"
        np.testing.assert_allclose(w_got[c], K.nets.pack(w64), err_msg=msg, **tol)
        if loop is not None:
            np.testing.assert_allclose(w_got[c], loop[0][c], err_msg=msg, **loop_tol)
        if not ch.loss:
            assert l_got[c] is None
            continue
        want = (ch.loss_init if ch.acc else 0.0) + float(l64)
        np.testing.assert_allclose(l_got[c], want, rtol=1e-4, err_msg=msg)
        if loop is not None:
            np.testing.assert_allclose(loop[1][c], want, rtol=1e-4, err_msg=msg)


def n_steps(K, E, T):
    steps = K.L.lib().rcmarl_minibatch_steps(E, T, MB)
    assert steps == E * (-(-T // MB))
    return steps


# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,E,T", [(1024, 10, 20), (1024, 10, 70), (4096, 2, 70)])
def test_trainer_chain_mix_matches_oracle_and_step_loop(K, N, E, T):
    """The 8 chains of [Cooperative, Malicious, Greedy, Cooperative, Malicious] in one launch.  T = 20 < 32: one short
    mini-batch per epoch (the trainer while its buffer holds fewer than 32 time rows); T = 70: 32 + 32 + 6 time rows."""
    rs = np.random.RandomState(N + E + T)
    buf = Buf(K, rs, N, T)
    chains = trainer_chains(K, rs, buf, MIXED)
    assert len(chains) == 8
    assert sum(not ch.loss for ch in chains) == 2 and sum(ch.stride == NA for ch in chains) == 1
    assert len({ch.lr(0.012) for ch in chains}) == 8
    n_steps(K, E, T)
    perms, dperm = perm_tables(K, rs, len(chains), E, T)
    got = run_persistent(K, buf, chains, dperm, E, 0.012, K.ops.MinibatchCells())
    loop = run_steps(K, buf, chains, dperm, E, 0.012)
    tol = ROUND if E == 10 else SHORT
    check_against_oracle(K, buf, chains, perms, E, 0.012, got, tol, loop, ROUND if E == 10 else SHORT_LOOP)


def test_max_jobs_chains_match_oracle_and_one_more_is_refused(K):
    """RCMARL_MAX_JOBS chains of all three input kinds, strided and contiguous targets, per-chain learning rates (the
    trainer sizes its cells for RCMARL_MAX_JOBS); a 33rd chain is refused before anything is launched."""
    rs = np.random.RandomState(32)
    N, T, E, lr = 512, 40, 2, 0.01
    buf = Buf(K, rs, N, T)
    chains = []
    for j in range(K.L.MAX_JOBS + 1):
        kind = (IN_S, IN_SA, IN_NS)[j % 3]
        if j % 4 == 3:
            tgt, dtgt, stride = buf.r[:, j % NA].copy(), buf.dr[:, j % NA], NA
        else:
            (tgt, dtgt), stride = random_target(K, rs, buf), 1
        chains.append(Chain(rs, kind, tgt, dtgt, stride, coef=0.004 + 0.0005 * (j % 7) if j % 5 else 0.0,
                            loss=j % 3 != 2, acc=j % 2, loss_init=0.5 if j % 2 else -3.0))
    perms, dperm = perm_tables(K, rs, len(chains), E, T)
    cells = K.ops.MinibatchCells()
    ws, losses, gj, aj = jobs(K, buf, chains, dperm)
    ga, sa = K.ops.job_array(K.L.GradJob, gj), K.ops.job_array(K.L.SgdJob, aj)
    before = [w.clone() for w in ws], cells.buf.clone()
    st = K.L.lib().rcmarl_minibatch_fit(C.byref(buf.rows(K, dperm)), ga, sa, len(chains), E, T, MB, lr,
                                        cells.buf.data_ptr(), cells.buf.numel(), cells.seq, K.ops._stream())
    torch.cuda.synchronize()
    assert st == ERR_ARG
    assert all(torch.equal(w, b) for w, b in zip(ws, before[0])) and torch.equal(cells.buf, before[1])

    chains, perms, dperm = chains[:K.L.MAX_JOBS], perms[:K.L.MAX_JOBS], dperm[:K.L.MAX_JOBS]
    got = run_persistent(K, buf, chains, dperm, E, lr, cells)
    loop = run_steps(K, buf, chains, dperm, E, lr)
    check_against_oracle(K, buf, chains, perms, E, lr, got, SHORT, loop, SHORT_LOOP)


def test_consecutive_fits_with_different_grids_share_cells(K, SMS):
    """Three fits in a row on one MinibatchCells: A (3 chains, N = 4096), B (1 chain over every SM, so its CTAs overwrite
    A's level-1 cells with another chain and slice layout), C (the 8-chain trainer mix, N = 1024).  Each fit matches the
    oracle and advances cells.seq by exactly its step count."""
    rs = np.random.RandomState(7)
    E, T, lr = 2, 40, 0.01
    cells = K.ops.MinibatchCells()
    big, small = Buf(K, rs, 4096, T), Buf(K, rs, 1024, T)
    fits = [("A", big, [Chain(rs, k, *random_target(K, rs, big)) for k in (IN_S, IN_SA, IN_S)]),
            ("B", big, [Chain(rs, IN_SA, *random_target(K, rs, big))]),
            ("C", small, trainer_chains(K, rs, small, MIXED))]
    plan = {name: grad_ctas(K, NA, [ch.kind for ch in chains], MSE, MB * buf.N, SMS, balanced=True)
            for name, buf, chains in fits}
    assert plan["B"] == [SMS]                         # one chain gets every SM
    assert plan["A"] != plan["B"] != plan["C"] and len(plan["C"]) == 8
    steps = n_steps(K, E, T)
    for name, buf, chains in fits:
        perms, dperm = perm_tables(K, rs, len(chains), E, T)
        seq0 = cells.seq
        got = run_persistent(K, buf, chains, dperm, E, lr, cells)
        assert cells.seq == seq0 + steps, name
        check_against_oracle(K, buf, chains, perms, E, lr, got, SHORT)


def test_ops_restarts_on_clean_cells_before_the_sequence_numbers_run_out(K):
    """ops.minibatch_fit zeroes the cells and restarts at 1 when a call would reach 0xFFFF0000: a 9-step fit from
    cells.seq = 0xFFFF0000 - 2 on cells used before gives the same bits as on fresh cells and leaves cells.seq = 10."""
    rs = np.random.RandomState(9)
    N, T, E, lr = 1024, 70, 3, 0.01
    assert n_steps(K, E, T) == 9
    buf = Buf(K, rs, N, T)
    chains = [Chain(rs, k, *random_target(K, rs, buf)) for k in (IN_S, IN_SA, IN_S)]
    perms, dperm = perm_tables(K, rs, len(chains), E, T)
    fresh = run_persistent(K, buf, chains, dperm, E, lr, K.ops.MinibatchCells(3, K.L.param_count(3 * NA, 1)))
    used = K.ops.MinibatchCells(3, K.L.param_count(3 * NA, 1))
    run_persistent(K, buf, chains, dperm, E, 2 * lr, used)          # other values in the cells
    assert used.seq == 10
    used.seq = 0xFFFF0000 - 2
    got = run_persistent(K, buf, chains, dperm, E, lr, used)
    assert used.seq == 10
    for c in range(len(chains)):
        assert np.array_equal(got[0][c], fresh[0][c]), c
        assert got[1][c] == fresh[1][c], c
    check_against_oracle(K, buf, chains, perms, E, lr, got, SHORT)


def test_c_abi_sequence_number_limits(K):
    """On freshly zeroed cells: seq_first = 0xFFFFFFFE - steps (the largest accepted) gives the bits of seq_first = 1;
    0xFFFFFFFF - steps and 0 are refused with RCMARL_ERR_ARG and change neither the weights nor the cells."""
    rs = np.random.RandomState(11)
    N, T, E, lr = 1024, 70, 3, 0.01
    steps = n_steps(K, E, T)
    buf = Buf(K, rs, N, T)
    chains = [Chain(rs, k, *random_target(K, rs, buf)) for k in (IN_SA, IN_S)]
    perms, dperm = perm_tables(K, rs, len(chains), E, T)

    def call(seq):
        cells = K.ops.MinibatchCells(len(chains), K.L.param_count(3 * NA, 1))
        ws, losses, gj, aj = jobs(K, buf, chains, dperm)
        before = [w.clone() for w in ws]
        st = K.L.lib().rcmarl_minibatch_fit(C.byref(buf.rows(K, dperm)), K.ops.job_array(K.L.GradJob, gj),
                                            K.ops.job_array(K.L.SgdJob, aj), len(chains), E, T, MB, lr,
                                            cells.buf.data_ptr(), cells.buf.numel(), seq, K.ops._stream())
        got = fetch(ws, losses)
        if st != OK:
            assert all(torch.equal(w, b) for w, b in zip(ws, before))
            assert not cells.buf.any()
        return st, got
    st1, first = call(1)
    st_max, last = call(SEQ_LIMIT - 1 - steps)
    assert st1 == OK and st_max == OK
    for c in range(len(chains)):
        assert np.array_equal(first[0][c], last[0][c]), c
        assert first[1][c] == last[1][c], c
    check_against_oracle(K, buf, chains, perms, E, lr, first, SHORT)
    assert call(SEQ_LIMIT - steps)[0] == ERR_ARG
    assert call(0)[0] == ERR_ARG


def test_c_abi_refuses_bad_arguments_without_launching(K, SMS):
    """Each malformed call returns its documented status and leaves the weights and the whole cells buffer bitwise
    unchanged.  Every buffer is real and full-size, so none of these calls could touch memory out of bounds even if it
    were accepted: one mini-batch (T < 32, E = 1), so a null time_idx would read the first rows in order; rows and weights
    with room for the 16-agent kernel; cells sized for it."""
    rs = np.random.RandomState(13)
    N, T, E, lr = 1024, 20, 1, 0.01
    buf = Buf(K, rs, N, T, room_for_16=True)
    chains = [Chain(rs, k, *random_target(K, rs, buf)) for k in (IN_S, IN_SA, IN_S)]
    kinds = [ch.kind for ch in chains]
    perms, dperm = perm_tables(K, rs, len(chains), E, T)
    cells = K.ops.MinibatchCells(len(chains), K.L.param_count(48, 1))
    ws, losses, gj, aj = jobs(K, buf, chains, dperm, room_for_16=True)
    ga, sa = K.ops.job_array(K.L.GradJob, gj), K.ops.job_array(K.L.SgdJob, aj)
    # the plan's cells: level 1 one row per CTA, level 2 two rows per chain, rows of (max n + 1) {value, seq} cells
    maxn = max(K.L.param_count(d_in(k), 1) for k in kinds) + 1
    need = (sum(grad_ctas(K, NA, kinds, MSE, T * N, SMS, balanced=True)) + 2 * len(chains)) * maxn * 8 + 64
    assert need <= cells.buf.numel()

    def call(rows=None, ga=ga, sa=sa, n_jobs=len(chains), epochs=E, nbytes=None):
        rows = buf.rows(K, dperm) if rows is None else rows
        st = K.L.lib().rcmarl_minibatch_fit(C.byref(rows), ga, sa, n_jobs, epochs, T, MB, lr, cells.buf.data_ptr(),
                                            cells.buf.numel() if nbytes is None else nbytes, cells.seq, K.ops._stream())
        torch.cuda.synchronize()
        return st

    assert call() == OK                               # cells and weights now hold a fit's values
    cells.seq += n_steps(K, E, T)
    w_before = [w.clone() for w in ws]
    c_before = cells.buf.clone()

    def edited(arr, cls, j, **fields):
        out = K.ops.job_array(cls, arr)
        for k, v in fields.items():
            setattr(out[j], k, v)
        return out
    other = _padded(K, ws[1].clone(), 2)
    rows7 = buf.rows(K, dperm)
    rows7.n_agents = 7
    cases = {
        "cells 8 bytes short of the plan": (ERR_WORKSPACE, dict(nbytes=need - 8)),
        "sgd dst is not the grad job's w": (ERR_ARG, dict(sa=edited(sa, K.L.SgdJob, 1, dst=other.data_ptr(),
                                                                    src=other.data_ptr()))),
        "first != 0": (ERR_ARG, dict(sa=edited(sa, K.L.SgdJob, 0, first=1))),
        "wrong n": (ERR_ARG, dict(sa=edited(sa, K.L.SgdJob, 2, n=sa[2].n - 1))),
        "null time_idx": (ERR_ARG, dict(ga=edited(ga, K.L.GradJob, 1, time_idx=None))),
        "epochs = 0": (ERR_ARG, dict(epochs=0)),
        "n_jobs = 0": (ERR_ARG, dict(n_jobs=0)),
        "n_agents = 7": (ERR_ARG, dict(rows=rows7)),
    }
    for name, (status, kw) in cases.items():
        assert call(**kw) == status, name
        assert all(torch.equal(w, b) for w, b in zip(ws, w_before)), name
        assert torch.equal(cells.buf, c_before), name
    assert call(nbytes=need) == OK                    # exactly the plan's size is enough
    assert not all(torch.equal(w, b) for w, b in zip(ws, w_before))
