"""GPU parity of nearest-neighbour mixing (rcmarl_nnm_mix, include/rcmarl.h) against the float64 oracle
(tests/nnm_oracle.py): the kernel at n_in 1..16 over every H, the trainer's parameter counts and repeated in-nodes,
32 jobs per launch, the mixing matrix, the bitwise consequences the header states (multi-Krum at H = 0, pass-through at
H = n - 1, rows of 1e30 / +-inf), bitwise determinism, the staging bound in a fresh process and the refusals; whole
update rounds through Trainer with a Byzantine agent and every cooperative agent mixing under each of the 8 rules, a
16-agent team where some cooperative agents mix, a world-1 PeerComm, and the per-agent API.

Selections are compared exactly where the oracle's relative distance gap at every row's n - H boundary is above 1e-4
(nnm_oracle.margin: a tie between identical rows, e.g. a repeated in-node, is exact in any precision and does not
count); the kernel's fp32 distances differ from the oracle's fp64 ones by far less.  Elsewhere each mixed row is checked
against the mean of the rows the kernel chose, and in update rounds the oracle follows the kernel's pick: the min-max
attack places its message at exactly the honest messages' largest distance in exact arithmetic, so those boundaries are
near ties that fp32 may break either way.
A mixed row's atol is 4e-6 max|x| (a mean of the chosen rows, as multi-Krum's); after whole update rounds weights rtol
1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as test_trainer_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import agg_oracle as AO                                # noqa: E402
import dnc_oracle as DO                                # noqa: E402
import nnm_oracle as NO                                # noqa: E402
import team_util as TU                                 # noqa: E402
import vector_oracle as VO                             # noqa: E402
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
C2_BYZ = ["Cooperative"] * 4 + ["Byzantine"]
ATTACKS = {"alie": 1.5, "minmax_uv": 1.0}
RULES = ("clip", "trim", "wmsr", "krum", "mkrum", "scclip", "gmed", "dnc")
PAR_COUNTS = (661, 761, 1101, 1421)                    # 5- / 16-agent critic / TR nets
EIG_GAP, SCORE_GAP = 1e-3, 1e-6                        # dnc's margins (test_dnc_gpu.py)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def out_atol(vmax):
    return 4e-6 * max(vmax, 1.0)


def nnm_job(K, dst, msgs, P, nodes, H, weights_out=None):
    """Mixed row k at dst + k * msgs.shape[1]."""
    return K.ops.vector_job(dst, msgs, msgs.shape[1], P, nodes, H, K.L.MIX_NNM, weights_out=weights_out)


# ---------------------------------------------------------------------------------------------------------- kernel
def _stack(rs, n_rows=24, P=max(PAR_COUNTS)):
    """Messages around a common centre (as trained networks are), each row with its own spread."""
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def _cases():
    """(n_in, H, P, repeated) over n_in 1..16 and every H in [0, n_in)."""
    return [(n_in, H, PAR_COUNTS[(n_in + H) % 4], (n_in + H) % 3 == 1 and n_in >= 3)
            for n_in in range(1, 17) for H in range(n_in)]


def _outputs(K, n_jobs, stride):
    return (torch.full((n_jobs, 16, stride), NAN, device=K.dev), torch.full((n_jobs, 256), NAN, device=K.dev))


def _jobs(K, rs, msgs, stack, cases, dst, wout):
    jobs, spec = [], []
    for j, (n_in, H, P, rep) in enumerate(cases):
        nodes = [int(x) for x in rs.choice(stack.shape[0], size=n_in, replace=False)]
        if rep:
            nodes[-1] = nodes[int(rs.randint(0, n_in - 1))]                     # a repeated in-node
        jobs.append(nnm_job(K, dst[j, 0], msgs, P, nodes, H, weights_out=wout[j]))
        spec.append((n_in, H, P, rep, nodes))
    return jobs, spec


def _check_rows_of_M(M, n_in, tag):
    for k in range(n_in):
        on = M[k] > 0
        assert on[k] and (M[k][on] == np.float32(1) / np.float32(on.sum())).all() and (M[k][~on] == 0).all(), tag


def test_nnm_mix_against_the_oracle(K):
    """n_in 1..16, every H, the trainer's parameter counts, repeated in-nodes, launches of 32 jobs: the mixed rows and M
    against the fp64 oracle, selections exactly where the gaps are clear."""
    rs = np.random.RandomState(5100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    S = stack.shape[1]
    cases = _cases()
    n_exact = 0
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        dst, wout = _outputs(K, len(part), S)
        jobs, spec = _jobs(K, rs, msgs, stack, part, dst, wout)
        K.ops.nnm_mix(jobs)
        got, gw = dst.cpu().numpy(), wout.cpu().numpy()
        for j, (n_in, H, P, rep, nodes) in enumerate(spec):
            X = stack[nodes, :P].astype(f64)
            tag = f"n_in={n_in} H={H} P={P} nodes={nodes}"
            assert np.isnan(got[j, n_in:]).all() and np.isnan(got[j, :n_in, P:]).all(), f"{tag}: wrote past the rows"
            assert np.isnan(gw[j, n_in * n_in:]).all(), f"{tag}: wrote past n_in^2 weights"
            M = gw[j, :n_in * n_in].reshape(n_in, n_in)
            _check_rows_of_M(M, n_in, tag)
            assert ((M > 0).sum(1) == n_in - H).all(), tag
            want, wM = NO.mix(X, H)
            if NO.clear(X, H):
                n_exact += 1
                np.testing.assert_array_equal(M, wM.astype(np.float32), err_msg=tag)
            else:                                     # an unclear selection: each row is the mean the kernel chose
                want = (M > 0).astype(f64) @ X / (M > 0).sum(1, keepdims=True)
            close(got[j, :n_in, :P], want, rtol=0, atol=out_atol(np.abs(X).max()), err_msg=tag)
    print(f"nnm jobs {len(cases)}, selections compared exactly {n_exact}")
    assert n_exact >= 0.8 * len(cases), n_exact


def test_bitwise_consequences(K):
    """H = 0: every mixed row is multi-Krum's output at H = 0, bit for bit (n_in >= 3), and M is its weights; H = n - 1:
    every row passes through; rows of 1e30 / +-inf pass through and no finite row mixes one in."""
    rs = np.random.RandomState(5200)
    stack = _stack(rs, n_rows=20)
    S = stack.shape[1]
    bad = {16: 1e30, 17: np.inf, 18: -np.inf, 19: -1e30}
    for r, v in bad.items():
        cols = np.arange(S) if r % 2 == 0 else np.arange(0, S, 3)
        stack[r, cols] = v
    msgs = to_dev(K, stack)[0]
    cases = []
    for n_in in range(3, 17):
        cases.append((n_in, 0, [int(x) for x in rs.choice(16, size=n_in, replace=False)]))
    for n_in in (1, 2, 5, 16):
        cases.append((n_in, n_in - 1, [int(x) for x in rs.choice(20, size=n_in, replace=False)]))
    for n_in, H, b in [(4, 1, [16]), (5, 2, [17, 18]), (8, 3, [19, 17, 16]), (16, 4, [16, 17, 18, 19]), (3, 1, [18])]:
        honest = [int(x) for x in rs.choice(np.arange(1, 16), size=n_in - 1 - len(b), replace=False)]
        cases.append((n_in, H, [0] + [int(x) for x in rs.permutation(honest + b)]))
    dst, wout = _outputs(K, len(cases), S)
    K.ops.nnm_mix([nnm_job(K, dst[j, 0], msgs, S, nodes, H, weights_out=wout[j]) for j, (_, H, nodes) in enumerate(cases)])
    mk = torch.full((len(cases), S), NAN, device=K.dev)
    mkw = torch.full((len(cases), 16), NAN, device=K.dev)
    zero = [j for j, (n_in, H, _) in enumerate(cases) if H == 0 and n_in >= 3]
    K.ops.vector_aggregate([K.ops.vector_job(mk[j], msgs, S, S, cases[j][2], 0, "mkrum", weights_out=mkw[j]) for j in zero])
    got, gw, mk, mkw = dst.cpu().numpy(), wout.cpu().numpy(), mk.cpu().numpy(), mkw.cpu().numpy()
    for j, (n_in, H, nodes) in enumerate(cases):
        M = gw[j, :n_in * n_in].reshape(n_in, n_in)
        tag = f"n_in={n_in} H={H} nodes={nodes}"
        if j in zero:
            for k in range(n_in):
                np.testing.assert_array_equal(got[j, k], mk[j], err_msg=tag)
                np.testing.assert_array_equal(M[k], mkw[j, :n_in], err_msg=tag)
        elif H == n_in - 1 and not any(x in bad for x in nodes):
            np.testing.assert_array_equal(got[j, :n_in], stack[nodes], err_msg=tag)
            np.testing.assert_array_equal(M, np.eye(n_in, dtype=np.float32), err_msg=tag)
        else:
            is_bad = np.array([x in bad for x in nodes])
            for k in np.flatnonzero(is_bad):
                np.testing.assert_array_equal(got[j, k], stack[nodes[k]], err_msg=tag)
                assert M[k, k] == 1
            assert (M[~is_bad][:, is_bad] == 0).all() and np.isfinite(got[j, :n_in][~is_bad]).all(), tag
            _check_rows_of_M(M, n_in, tag)
            X = stack[nodes].astype(f64)
            if NO.clear(X, H):
                np.testing.assert_array_equal(M, NO.mix(X, H)[1].astype(np.float32), err_msg=tag)
            for k in np.flatnonzero(~is_bad):                # each finite row: the mean of the rows the kernel chose
                close(got[j, k], X[M[k] > 0].mean(0), rtol=0, atol=out_atol(np.abs(X[~is_bad]).max()), err_msg=tag)


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(5300)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases()[::4][:32]
    dst, wout = _outputs(K, len(cases), stack.shape[1])
    jobs, _ = _jobs(K, rs, msgs, stack, cases, dst, wout)
    assert len(jobs) == len(cases) >= 30 and {c[0] for c in cases} >= {1, 4, 16}

    def run(groups):
        dst.fill_(NAN)
        wout.fill_(NAN)
        for g in groups:
            K.ops.nnm_mix(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(wout, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(5400)
    P = 700
    stack = _stack(rs, n_rows=8, P=P)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((3, 4, P), NAN, device=K.dev)
    wout = torch.full((3, 256), NAN, device=K.dev)
    V = K.ops.vector_job
    X = K.L.MIX_NNM
    good = V(dst[0, 0], msgs, P, P, [0, 1, 2, 3], 1, X, weights_out=wout[0])
    d, w = dst[1, 0], wout[1]
    bad = [V(d, msgs, P, P, [0, 1, 2], 3, X, weights_out=w),                    # H >= n_in
           V(d, msgs, P, P, [0, 1, 2], -1, X, weights_out=w),
           V(d, msgs, P, P, [], 0, X, weights_out=w),
           V(d, msgs, P, P, list(range(8)) * 2 + [0], 0, X, weights_out=w),     # 17 in-nodes
           V(d, msgs, P, P, [0, -1, 2], 0, X, weights_out=w),
           V(d, msgs, P, P, [0, 1, 2], 0, 1, weights_out=w),                    # not the nnm rule
           V(d, msgs, P, 0, [0, 1, 2], 0, X, weights_out=w),
           V(msgs[2], msgs, P, P, [0, 1, 2], 0, X, weights_out=w),              # dst row 0 is an in-node row
           V(msgs[5], msgs, P, P, [0, 1, 2, 6], 0, X, weights_out=w),           # dst row 1 is in-node row 6
           V(dst[0, 2], msgs, P, P, [5, 6, 7], 0, X, weights_out=w),            # dst rows on the other job's
           V(d, msgs, P, 48 * 1024 // 3 + 1, [0, 1, 2], 0, X, weights_out=w),   # over the shared-memory staging limit
           V(d, msgs, P, P, [0, 1, 2], 0, X, weights_out=msgs[1][5:]),          # weights_out on an in-node row
           V(d, msgs, P, P, [0, 1, 2], 0, X, weights_out=dst[0, 3][10:]),       # ... on the other job's dst row 3
           V(d, msgs, P, P, [0, 1, 2], 0, X, weights_out=dst[1, 1][3:]),        # ... on its own dst row 1
           V(d, msgs, P, P, [0, 1, 2], 0, X, weights_out=wout[0][15:]),         # ... on the other's weights_out
           V(d, msgs, P // 2, P // 2 + 1, [0, 1, 2], 0, X, weights_out=w)]      # its own dst rows overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.nnm_mix([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(wout).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.nnm_mix([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(wout).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.nnm_mix([good])
    assert torch.isfinite(dst[0]).all() and torch.isfinite(wout[0, :16]).all() and torch.isnan(dst[1:]).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import nnm_oracle as NO
rs = np.random.RandomState(5600)
for n_in, P in ((4, 3072), (16, 3072)):     # n_in * P = 12288 floats (48 KB), then the limit
    X = (rs.randn(n_in, P) * rs.uniform(0.1, 1, size=(n_in, 1)) + rs.randn(P)).astype(np.float32)
    msgs = torch.as_tensor(X).cuda()
    dst = torch.full((n_in, P), float("nan"), device="cuda")
    w = torch.full((n_in * n_in,), float("nan"), device="cuda")
    ops.nnm_mix([ops.vector_job(dst, msgs, P, P, list(range(n_in)), 1, L.MIX_NNM, weights_out=w)])
    M = w.cpu().numpy().reshape(n_in, n_in)
    assert ((M > 0).sum(1) == n_in - 1).all(), M
    want = (M > 0).astype(np.float64) @ X.astype(np.float64) / (n_in - 1)
    err = float(np.abs(dst.cpu().numpy() - want).max())
    assert err < 4e-6 * np.abs(X).max(), (n_in, P, err)
    assert not NO.clear(X.astype(np.float64), 1) or (M == NO.mix(X.astype(np.float64), 1)[1].astype(np.float32)).all()
print("ok")
"""


def test_staging_limit_as_the_first_launch_of_a_process(K, tmp_path):
    """Static shared memory counts against the default 48 KB too: a job of n_in * n = 12288 floats (48 KB of dynamic
    staging) runs as the first nnm launch of a fresh process, as does one at RCMARL_NNM_MAX_FLOATS."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    assert 4 * 3072 == 12288 and 16 * 3072 == K.L.NNM_MAX_FLOATS
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
class DncAgent(DO.RPBCACOracleAgent):
    """The dnc oracle agent, following the kernel's selection where the oracle's margins are not clear.  Mixed messages
    repeat (at n_in = 4 and H = 1 each is the mean of 3 of the 4), and repeated rows give repeated eigenvalues or equal
    scores, where the selection is not a property of the messages (include/rcmarl.h).  kernel_w[epoch] = [critic w, TR
    w] of the agent's dnc job; the agent makes 4 aggregations per epoch (critic, TR hidden; critic, TR estimates)."""

    kernel_w = None

    def _aggregate(self, w, msgs):
        X = np.stack([DO.AT.pack(m, self.dtype) for m in msgs])
        eig, gap = DO.margins(X, self.H)
        c = len(self.last_weights)
        if (eig < EIG_GAP or gap < SCORE_GAP) and self.kernel_w is not None:
            keep = self.kernel_w[c // 4][c % 2][:X.shape[0]] > 0
            wt = keep / keep.sum()
            self.last_weights.append(wt)
            self.last_margins.append((eig, gap))
            return DO.AT.unpack(X[keep].sum(0) / keep.sum(), w)
        return super()._aggregate(w, msgs)


def _oracle_agent(rule, w, fast, gamma, H):
    cls = DncAgent if rule == "dnc" else VO.RPBCACOracleAgent if rule in VO.RULES else AO.RPBCACOracleAgent
    return cls(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, aggregation=rule)


def _follow_dnc(agents, runs):
    """Give each dnc oracle agent the kernel's dnc weights of epoch e from runs[e] (a Trainer whose last epoch is e)."""
    for i, ag in enumerate(agents):
        if isinstance(ag, DncAgent):
            ag.kernel_w = [[tr.dnc_weights[2 * tr.dnc_agents.index(i) + t].cpu().numpy() for t in range(2)]
                           for tr in runs]


def _perms():
    """The same mini-batch permutations, call by call, for every run."""
    rs = np.random.RandomState(1700)
    return lambda T_: rs.permutation(T_)


def _trainer_round(cfg, rows, round_, n_epochs, mixing):
    from rcmarl.trainer import Trainer
    tr = Trainer(n_epochs=n_epochs, mixing=mixing, perm_source=_perms(), **cfg)
    tr.load_rows(*rows)
    tr.episodes_done = round_
    return tr, tr.update_round()


def _kernel_M(cfg, rows, round_, mixing):
    """(Trainer after a two-epoch round, its losses, {epoch: Trainer.mixing_matrices()}, [the one-epoch Trainer, the
    two-epoch one]): epoch 0's from a one-epoch round from the same state, which runs the same launches bit for bit."""
    tr1, _ = _trainer_round(cfg, rows, round_, 1, mixing)
    tr, got = _trainer_round(cfg, rows, round_, 2, mixing)
    return tr, got, {0: tr1.mixing_matrices(), 1: tr.mixing_matrices()}, [tr1, tr]


def _oracle_round(agents, labels, in_nodes, rows, attacks, mixing, H, N, T, round_, kernel_M, seed=0, n_epochs=2):
    log = {}
    hook = NO.mixing_hook(labels, in_nodes, mixing, H, inner=AA.make_hook(labels, in_nodes, attacks, seed=seed,
                                                                          round_=round_), log=log, kernel_M=kernel_M)
    loss = NO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=_perms(), messages_hook=hook)
    return loss, log


def _check_mixing(tr, agents, rules, log):
    """Trainer.mixing_matrices against the oracle's last-epoch M where the selections are clear, and
    neighbour_weights (the effective w M) of the whole-message rules.  Returns how many M were compared exactly."""
    mats = tr.mixing_matrices()
    assert sorted(mats) == sorted(log) == tr.mix_agents
    n_exact = 0
    clear = {}
    for i, M in mats.items():
        n_in = len(tr.in_nodes[i])
        for t in range(2):
            wM, _, clear[i, t] = log[i][-1][t]
            _check_rows_of_M(M[t], n_in, f"agent {i} net {t}")
            if clear[i, t]:
                n_exact += 1
            np.testing.assert_array_equal(M[t], wM.astype(np.float32), err_msg=f"agent {i} net {t}")
    got = tr.neighbour_weights()
    whole = VO.RULES + ("dnc",)
    assert sorted(got) == [i for i in tr.coop if rules[i] in whole]
    for i, w in got.items():
        if i not in mats:
            continue
        rule_w = np.stack(agents[i].last_weights[-4:-2])                 # the last epoch's critic and TR aggregations
        for t in range(2):
            if not clear[i, t]:
                continue
            want = rule_w[t] @ log[i][-1][t][0]
            if rules[i] == "dnc":
                if all(m >= g for m, g in zip(agents[i].last_margins[-4 + t], (EIG_GAP, SCORE_GAP))):
                    close(w[t], want, rtol=1e-6, atol=1e-7, err_msg=f"agent {i} net {t}")
            elif rules[i] in ("krum", "mkrum"):
                close(w[t], want, rtol=1e-6, atol=1e-7, err_msg=f"agent {i} net {t}")
            else:
                close(w[t], want, rtol=0, atol=2e-3, err_msg=f"agent {i} net {t}")
            np.testing.assert_allclose(w[t].sum(), 1.0, atol=1e-5)
    return n_exact


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("kind", list(ATTACKS))
@pytest.mark.parametrize("rule", RULES)
def test_c2_update_round_with_a_byzantine_agent(K, rule, kind, N):
    """The benchmark's 5-agent team with agent 4 Byzantine, every cooperative agent mixing before `rule` (H = 1): one
    update round of two epochs against the oracle's round with the attack hook inside the mixing hook; one nnm launch
    per epoch more than without mixing."""
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(5500 + N)
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule)
    tr, got, kernel_M, runs = _kernel_M(cfg, rows, round_, "nnm")
    agents = [_oracle_agent(rule, w[i], 0.01, gamma, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    _follow_dnc(agents, runs)
    want, log = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: attack}, ["nnm"] * 4 + [None], [1] * 5, N, T, round_,
                              kernel_M, seed=9)
    n_exact = _check_mixing(tr, agents, [rule] * 4 + [None], log)
    print(f"{rule} {kind} N={N}: last-epoch M clear (compared with the oracle's own) {n_exact} of 8")
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    plain, _ = _trainer_round(cfg, rows, round_, 2, None)
    assert plain.mixing_matrices() == {}
    assert tr.launches - plain.launches == 2                                    # one nnm launch per epoch
    assert tr.msg_c.shape[0] - plain.msg_c.shape[0] == 4 * 4                    # n_in mixed rows per agent


RULES16 = ["dnc", "clip", "gmed", "trim", "mkrum", "wmsr", "scclip", "krum"]   # the 8 cooperative agents, in order
MIX16 = ["nnm", None, "nnm", "nnm", None, "nnm", "nnm", "nnm"]


def test_16_agent_team_where_some_agents_mix(K):
    """16 agents (8 cooperative, 5 Byzantine with mixed attacks, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, one
    receiver listing a Byzantine agent twice) with the cooperative agents' rules and mixing set per agent."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mixing = ["clip"] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mixing[i] = RULES16[q], MIX16[q]
    H = [max(h, 1) if rules[i] == "dnc" else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(_oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[attacks.get(i) for i in range(16)])
    tr, got, kernel_M, runs = _kernel_M(cfg, rows, round_, mixing)
    _follow_dnc(agents, runs)
    want, log = _oracle_round(agents, labels, in_nodes, rows, attacks, mixing, H, N, T, round_, kernel_M, seed=4)
    assert len(tr.mix_agents) == 6 and tr.msg_c.shape[0] == 16 + len(tr.byz_pairs) + 4 + 1 + 6 * 8
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]}, {mixing[i]})")
    n_exact = _check_mixing(tr, agents, rules, log)
    print(f"16 agents: M compared exactly {n_exact} of {2 * len(tr.mix_agents)}")


@pytest.fixture
def gloo_world1(tmp_path):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'pg'}", rank=0, world_size=1,
                            timeout=datetime.timedelta(seconds=120))
    made = []
    yield made
    for c in made:
        c.close()
    dist.destroy_process_group()


def _state(tr):
    return [getattr(tr, n).clone() for n in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v", "vec_weights",
                                             "dnc_weights", "mix_weights", "msg_c", "msg_t")]


def test_world1_peer_comm_with_mixing_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents mix."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["dnc", "mkrum", "trim", "clip", "clip"], mixing=["nnm", "nnm", "nnm", None, None],
                     attack=("minmax_std", 1.0))
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append(_state(tr))
    assert all(torch.equal(x, y) for x, y in zip(*runs))


# ---------------------------------------------------------------------------------------------------------- agent API
@pytest.mark.parametrize("rule", ["clip", "mkrum"])
def test_rpbcac_agent_methods_with_mixing(K, rule):
    """RPBCAC_agent(..., mixing="nnm"): hidden consensus, estimate consensus, projection step and
    _resilient_aggregation against the oracle agent fed the oracle's mixed messages."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H = 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule, mixing="nnm")
    ora = _oracle_agent(rule, w[0], 0.01, 0.9, H)
    nbrs = [0, 1, 3, 2, 4]
    cmsgs = [list(w[j][1]) for j in nbrs]
    tmsgs = [list(w[j][2]) for j in nbrs]
    hook = NO.mixing_hook(["Cooperative"], [[0]], ["nnm"], [H], inner=lambda e, c, t: ({0: c}, {0: t}))
    mc, mt = hook(0, cmsgs, tmsgs)
    mc, mt = mc[0], mt[0]
    for msgs in (cmsgs, tmsgs):
        X = np.stack([np.concatenate([np.asarray(x, f64).ravel() for x in m]) for m in msgs])
        assert NO.clear(X, H), NO.margin(X, H)
    ag.resilient_consensus_critic_hidden(cmsgs)
    ag.resilient_consensus_TR_hidden(tmsgs)
    ora.resilient_consensus_critic_hidden(mc)
    ora.resilient_consensus_TR_hidden(mt)
    for k in range(6):
        close(ag.critic.get_weights()[k], ora.critic[k], rtol=1e-4, atol=1e-5)
        close(ag.TR.get_weights()[k], ora.TR[k], rtol=1e-4, atol=1e-5)
    cagg, tagg = ag.resilient_consensus_critic(s, cmsgs), ag.resilient_consensus_TR(sa, tmsgs)
    wc, wt = ora.resilient_consensus_critic(s, mc), ora.resilient_consensus_TR(sa, mt)
    close(cagg.numpy(), wc, rtol=1e-4, atol=1e-5)
    close(tagg.numpy(), wt, rtol=1e-4, atol=1e-5)
    ag.critic_update_team(s, cagg)
    ag.TR_update_team(sa, tagg)
    ora.critic_update_team(s, wc)
    ora.TR_update_team(sa, wt)
    for k in range(6):
        close(ag.critic.get_weights()[k], ora.critic[k], rtol=1e-4, atol=1e-5)
        close(ag.TR.get_weights()[k], ora.TR[k], rtol=1e-4, atol=1e-5)
    rs = np.random.RandomState(1500)
    v = rs.randn(7, 3, 11).astype(np.float32) * rs.uniform(0.2, 2, size=(7, 1, 1)).astype(np.float32)
    v[5, 1] = np.inf
    for H_ in (2, 3):
        ag.H = H_
        X = v.reshape(7, -1).astype(f64)
        assert NO.clear(X, H_)
        Y, _ = NO.mix(X, H_)
        want = (AO.resilient_aggregation(Y, H_, "clip") if rule == "clip" else VO.aggregate(Y, H_, rule)[0])
        close(ag._resilient_aggregation(v).numpy(), want.reshape(3, 11), rtol=0,
              atol=out_atol(np.abs(v[np.isfinite(v)]).max()))
    with pytest.raises(K.L.RcmarlError):
        ag.H = 7
        ag._resilient_aggregation(v)
