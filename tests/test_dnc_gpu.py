"""GPU parity of the divide-and-conquer rule (rcmarl_dnc_aggregate, include/rcmarl.h) against the float64 oracle
(tests/dnc_oracle.py): the kernel at n_in 1..16 over the allowed H range, the trainer's parameter counts and repeated
in-nodes, 32 jobs per launch, weights_out, Byzantine rows of 1e30 / +-inf, bitwise determinism, the staging bound in a
fresh process and the refusals; whole update rounds through Trainer with a Byzantine agent, a 16-agent team mixing dnc
with coordinate-wise and distance-based rules, a world-1 PeerComm, and the per-agent API.

Selections are compared exactly where the oracle's margins are clear: a relative eigengap of at least 1e-3 and a
relative score gap at the removal boundary of at least 1e-6.  The kernel's Gram matrix is fp64 from the same fp32
inputs as the oracle's, so its scores differ from the oracle's by the rounding of the eigen-solvers only, far below
those gaps.  Elsewhere the kernel's aggregate is checked against the mean of the rows it kept.  The aggregate atol is
4e-6 max|x| (a mean of kept rows, as multi-Krum's); after whole update rounds weights rtol 1e-3 / atol 5e-5 and losses
rtol 2e-3 / atol 2e-5 (as test_trainer_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import agg_oracle as AO                                # noqa: E402
import dnc_oracle as DO                                # noqa: E402
import team_util as TU                                 # noqa: E402
import vector_oracle as VO                             # noqa: E402
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
C2_BYZ = ["Cooperative"] * 4 + ["Byzantine"]
ATTACKS = {"alie": 1.5, "ipm": 0.5, "gauss": 0.3, "minmax_uv": 1.0}
PAR_COUNTS = (661, 761, 1101, 1421)                    # 5- / 16-agent critic / TR nets
EIG_GAP, SCORE_GAP = 1e-3, 1e-6


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def out_atol(vmax):
    return 4e-6 * max(vmax, 1.0)


def clear(X, H):
    eig, gap = DO.margins(X, H)
    return eig >= EIG_GAP and gap >= SCORE_GAP


def dnc_job(K, dst, msgs, P, nodes, H, weights_out=None):
    return K.ops.vector_job(dst, msgs, msgs.shape[1], P, nodes, H, K.L.SPECTRAL_DNC, weights_out=weights_out)


# ---------------------------------------------------------------------------------------------------------- kernel
def _stack(rs, n_rows=24, P=max(PAR_COUNTS)):
    """Messages around a common centre (as trained networks are), each row with its own spread."""
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def _cases():
    """(n_in, H, P, repeated) over n_in 1..16 and H at the ends and the middle of [0, n_in)."""
    out = []
    for n_in in range(1, 17):
        for t, H in enumerate(sorted({0, (n_in - 1) // 2, n_in - 1})):
            out.append((n_in, H, PAR_COUNTS[(n_in + t) % 4], (n_in + t) % 2 == 1 and n_in >= 3))
    return out


def _jobs(K, rs, msgs, stack, cases, dst, wout):
    jobs, spec = [], []
    for j, (n_in, H, P, rep) in enumerate(cases):
        nodes = [int(x) for x in rs.choice(stack.shape[0], size=n_in, replace=False)]
        if rep:
            nodes[-1] = nodes[int(rs.randint(0, n_in - 1))]                     # a repeated in-node
        jobs.append(dnc_job(K, dst[j], msgs, P, nodes, H, weights_out=wout[j]))
        spec.append((n_in, H, P, rep, nodes))
    return jobs, spec


def test_dnc_aggregate_against_the_oracle(K):
    """n_in 1..16, H over its range, the trainer's parameter counts, repeated in-nodes, launches of 32 jobs: the
    aggregate and weights_out against the fp64 oracle, selections exactly where the margins are clear."""
    rs = np.random.RandomState(4100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases()
    n_exact = 0
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
        wout = torch.full((len(part), 16), NAN, device=K.dev)
        jobs, spec = _jobs(K, rs, msgs, stack, part, dst, wout)
        K.ops.dnc_aggregate(jobs)
        got, gw = dst.cpu().numpy(), wout.cpu().numpy()
        for j, (n_in, H, P, rep, nodes) in enumerate(spec):
            X = stack[nodes, :P].astype(f64)
            want, ww = DO.aggregate(X, H)
            tag = f"n_in={n_in} H={H} P={P} nodes={nodes}"
            assert np.isnan(got[j, P:]).all() and np.isnan(gw[j, n_in:]).all(), f"{tag}: wrote past n / n_in"
            kept = gw[j, :n_in] > 0
            assert kept.sum() == n_in - H, tag
            assert (gw[j, :n_in][kept] == np.float32(1) / np.float32(n_in - H)).all(), tag
            if clear(X, H):
                n_exact += 1
                np.testing.assert_array_equal(kept, ww > 0, err_msg=tag)
            else:                                    # an unclear selection: the kernel's is the mean it wrote
                want = X[kept].mean(0)
            close(got[j, :P], want, rtol=0, atol=out_atol(np.abs(X).max()), err_msg=tag)
    print(f"dnc jobs {len(cases)}, selections compared exactly {n_exact}")
    assert n_exact >= 0.8 * len(cases), n_exact


def test_byzantine_rows_get_weight_zero(K):
    """Rows holding +-inf (whole, or in some coordinates) and one row of +-1e30, at most H of them, with at least three
    unflagged rows, get weight 0; the aggregate is finite and matches the oracle."""
    rs = np.random.RandomState(4200)
    stack = _stack(rs, n_rows=20)
    P = stack.shape[1]
    huge = {16: 1e30, 19: -1e30}
    infs = {17: np.inf, 18: -np.inf}
    for r, v in {**huge, **infs}.items():
        cols = rs.choice(P, size=P // 3, replace=False) if r % 2 else np.arange(P)
        stack[r, cols] = v
    msgs = to_dev(K, stack)[0]
    cases = []
    for n_in, H, bad in [(4, 1, [16]), (5, 2, [17, 18]), (6, 3, [19, 17, 18]), (9, 3, [16, 18]), (16, 4, [19, 17]),
                         (16, 7, [16, 17, 18]), (3, 1, [19]), (12, 5, [17])]:
        honest = [int(x) for x in rs.choice(np.arange(1, 16), size=n_in - 1 - len(bad), replace=False)]
        nodes = [0] + [int(x) for x in rs.permutation(honest + bad)]                  # own (row 0) is honest
        cases.append((n_in, H, nodes))
    dst = torch.full((len(cases), P), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    K.ops.dnc_aggregate([dnc_job(K, dst[j], msgs, P, nodes, H, weights_out=wout[j])
                         for j, (n_in, H, nodes) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (n_in, H, nodes) in enumerate(cases):
        X = stack[nodes].astype(f64)
        want, ww = DO.aggregate(X, H)
        is_bad = np.array([k in huge or k in infs for k in nodes])
        assert np.isfinite(got[j]).all(), nodes
        assert (gw[j, :n_in][is_bad] == 0).all() and (ww[is_bad] == 0).all(), (nodes, gw[j, :n_in])
        if clear(X, H):
            np.testing.assert_array_equal(gw[j, :n_in] > 0, ww > 0, err_msg=str(nodes))
        else:
            want = X[gw[j, :n_in] > 0].mean(0)
        close(got[j], want, rtol=0, atol=out_atol(np.abs(X[~is_bad]).max()), err_msg=str(nodes))
    # every row flagged: the own row, weight e_0
    d, w = torch.full((P,), NAN, device=K.dev), torch.full((16,), NAN, device=K.dev)
    K.ops.dnc_aggregate([dnc_job(K, d, msgs, P, [17, 18, 17], 1, weights_out=w)])
    np.testing.assert_array_equal(d.cpu().numpy(), stack[17])
    np.testing.assert_array_equal(w.cpu().numpy()[:3], [1, 0, 0])


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(4300)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases()[::2][:32]
    dst = torch.full((len(cases), stack.shape[1]), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    jobs, _ = _jobs(K, rs, msgs, stack, cases, dst, wout)
    assert len(jobs) == len(cases) >= 20 and {c[0] for c in cases} >= {1, 4, 16}

    def run(groups):
        dst.fill_(NAN)
        wout.fill_(NAN)
        for g in groups:
            K.ops.dnc_aggregate(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(wout, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_dst_and_weights_untouched(K):
    rs = np.random.RandomState(4400)
    stack = _stack(rs, n_rows=8, P=700)
    msgs = to_dev(K, stack)[0]
    P = 700
    dst = torch.full((3, P), NAN, device=K.dev)
    wout = torch.full((3, 16), NAN, device=K.dev)
    V = K.ops.vector_job
    D = K.L.SPECTRAL_DNC
    good = V(dst[0], msgs, P, P, [0, 1, 2, 3], 1, D, weights_out=wout[0])
    d, w = dst[1], wout[1]
    bad = [V(d, msgs, P, P, [0, 1, 2], 3, D, weights_out=w),                    # H >= n_in
           V(d, msgs, P, P, [0, 1, 2], -1, D, weights_out=w),
           V(d, msgs, P, P, [], 0, D, weights_out=w),
           V(d, msgs, P, P, list(range(8)) * 2 + [0], 0, D, weights_out=w),     # 17 in-nodes
           V(d, msgs, P, P, [0, -1, 2], 0, D, weights_out=w),
           V(d, msgs, P, P, [0, 1, 2], 0, 1, weights_out=w),                    # not the dnc rule
           V(d, msgs, P, 0, [0, 1, 2], 0, D, weights_out=w),
           V(msgs[2], msgs, P, P, [0, 1, 2], 0, D, weights_out=w),              # dst is an in-node row
           V(msgs[3][3:], msgs, P, P, [5, 6, 7], 0, D, weights_out=w),          # dst overlaps a row of the other job
           V(d, msgs, P, 48 * 1024 // 5 + 1, [0, 1, 2], 0, D, weights_out=w),   # over the shared-memory staging limit
           V(d, msgs, P, P, [0, 1, 2], 0, D, weights_out=msgs[1][5:]),          # weights_out on an in-node row
           V(d, msgs, P, P, [0, 1, 2], 0, D, weights_out=dst[0][10:]),          # ... on the other job's dst
           V(d, msgs, P, P, [0, 1, 2], 0, D, weights_out=wout[0][3:]),          # ... on its weights_out
           V(dst[0][1:], msgs, P, P - 1, [0, 1, 2], 0, D, weights_out=w)]       # two dsts overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.dnc_aggregate([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(wout).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.dnc_aggregate([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(wout).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.dnc_aggregate([good])
    assert torch.isfinite(dst[0]).all() and torch.isnan(dst[1:]).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import dnc_oracle as DO
rs = np.random.RandomState(4600)
for n_in, P in ((4, 2048), (14, 3072)):     # (n_in + 2) * P = 12288 floats (48 KB), then the limit
    X = (rs.randn(n_in, P) * rs.uniform(0.1, 1, size=(n_in, 1)) + rs.randn(P)).astype(np.float32)
    msgs = torch.as_tensor(X).cuda()
    dst = torch.full((P,), float("nan"), device="cuda")
    w = torch.full((n_in,), float("nan"), device="cuda")
    ops.dnc_aggregate([ops.vector_job(dst, msgs, P, P, list(range(n_in)), 1, L.SPECTRAL_DNC, weights_out=w)])
    kept = w.cpu().numpy() > 0
    assert kept.sum() == n_in - 1, kept
    want = X[kept].astype(np.float64).mean(0)
    err = float(np.abs(dst.cpu().numpy() - want).max())
    assert err < 4e-6 * np.abs(X).max(), (n_in, P, err)
    _, ww = DO.aggregate(X.astype(np.float64), 1)
    eig, gap = DO.margins(X.astype(np.float64), 1)
    assert (eig < 1e-3 or gap < 1e-6) or (kept == (ww > 0)).all(), (kept, ww)
print("ok")
"""


def test_staging_limit_as_the_first_launch_of_a_process(K, tmp_path):
    """Static shared memory counts against the default 48 KB too: a job of (n_in + 2) * n = 12288 floats (48 KB of
    dynamic staging) runs as the first dnc launch of a fresh process, as does one at RCMARL_DNC_MAX_FLOATS."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    assert 6 * 2048 == 12288 and 16 * 3072 == K.L.DNC_MAX_FLOATS
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
def _c2_agents(w, gamma, H=1):
    ags = [DO.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, H=H, dtype=f64) for i in range(4)]
    ags.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    return ags


def _oracle_round(agents, labels, in_nodes, rows, attacks, N, T, round_, seed=0, n_epochs=2):
    prs = np.random.RandomState(1700)
    used = []

    def rec(T_):
        p = prs.permutation(T_)
        used.append(p)
        return p
    hook = AA.make_hook(labels, in_nodes, attacks, seed=seed, round_=round_)
    loss = DO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=rec, messages_hook=hook)
    return loss, used


def _check_neighbour_weights(tr, agents, rules):
    got = tr.neighbour_weights()
    whole = VO.RULES + ("dnc",)
    assert sorted(got) == [i for i, r in enumerate(rules) if r in whole and tr.labels[i] == "Cooperative"]
    n_sel = 0
    for i, w in got.items():
        want = np.stack(agents[i].last_weights[-4:-2])              # the last epoch's critic and TR aggregations
        if rules[i] == "dnc":
            for t in range(2):
                if all(m >= g for m, g in zip(agents[i].last_margins[-4 + t], (EIG_GAP, SCORE_GAP))):
                    n_sel += 1
                    np.testing.assert_array_equal(w[t] > 0, want[t] > 0, err_msg=f"agent {i} net {t}")
                    close(w[t], want[t], rtol=1e-6, atol=0, err_msg=f"agent {i} net {t}")
        elif rules[i] in ("krum", "mkrum"):
            np.testing.assert_array_equal(w > 0, want > 0, err_msg=f"agent {i}")
            close(w, want, rtol=1e-6, atol=0, err_msg=f"agent {i}")
        else:
            close(w, want, rtol=0, atol=2e-3, err_msg=f"agent {i}")
    return n_sel


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("kind", list(ATTACKS))
def test_c2_update_round_with_a_byzantine_agent(K, kind, N):
    """The benchmark's 5-agent team with agent 4 Byzantine, every cooperative agent on dnc (H = 1): one update round of
    two epochs against the oracle's round with the per-receiver hook; one dnc launch per epoch more than on clip."""
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(4500 + N)
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    agents = _c2_agents(w, gamma)
    want, used = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: attack}, N, T, round_, seed=9)
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=9, attack=attack)
    launches = []
    for agg in ("dnc", "clip"):
        it = iter(list(used))
        tr = Trainer(aggregation=agg, perm_source=lambda T_: next(it), **cfg)
        tr.load_rows(*rows)
        tr.episodes_done = round_
        got = tr.update_round()
        launches.append(tr.launches)
        if agg == "dnc":
            assert next(it, None) is None and tr.msg_c.shape[0] == 5 + 3 + 4
            for k in ("critic_loss", "TR_loss", "actor_loss"):
                np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
            for i in range(5):
                TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
            n_sel = _check_neighbour_weights(tr, agents, ["dnc"] * 4 + [None])
            assert n_sel >= 4, n_sel
        else:
            assert tr.neighbour_weights() == {} and tr.msg_c.shape[0] == 5 + 3
    assert launches[0] - launches[1] == 2                                       # one dnc launch per epoch


RULES16 = ["dnc", "clip", "gmed", "dnc", "mkrum", "wmsr", "dnc", "trim"]   # the 8 cooperative agents, in order


def test_16_agent_team_mixing_dnc_with_coordinate_and_vector_rules(K):
    """16 agents (8 cooperative, 5 Byzantine with mixed attacks, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, one
    receiver listing a Byzantine agent twice) with the cooperative agents' rules mixed per agent, dnc among them."""
    from rcmarl.trainer import Trainer
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules = ["clip"] * 16
    for q, i in enumerate(coop):
        rules[i] = RULES16[q]
    H = [max(h, 1) if rules[i] == "dnc" else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            cls = (DO.RPBCACOracleAgent if rules[i] == "dnc" else VO.RPBCACOracleAgent if rules[i] in VO.RULES
                   else AO.RPBCACOracleAgent)
            agents.append(cls(w[i][0], w[i][1], w[i][2], 0.002, fast[i], gamma, H=H[i], dtype=f64, aggregation=rules[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    want, used = _oracle_round(agents, labels, in_nodes, rows, attacks, N, T, round_, seed=4)
    it = iter(list(used))
    tr = Trainer(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
                 H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=4,
                 aggregation=rules, attack=[attacks.get(i) for i in range(16)], perm_source=lambda T_: next(it))
    tr.load_rows(*rows)
    tr.episodes_done = round_
    got = tr.update_round()
    assert next(it, None) is None
    assert tr.msg_c.shape[0] == 16 + len(tr.byz_pairs) + 2 + 3 and len(tr.dnc_agents) == 3
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]})")
    _check_neighbour_weights(tr, agents, rules)


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
                                             "dnc_weights")]


def test_world1_peer_comm_with_dnc_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents use dnc."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["dnc", "mkrum", "dnc", "clip", "clip"], attack=("minmax_std", 1.0))
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
def test_rpbcac_agent_methods_with_dnc(K):
    """RPBCAC_agent(..., aggregation="dnc"): hidden consensus, estimate consensus, projection step and
    _resilient_aggregation against the oracle agent."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H = 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation="dnc")
    ora = DO.RPBCACOracleAgent(w[0][0], w[0][1], w[0][2], 0.002, 0.01, 0.9, H=H, dtype=f64)
    nbrs = [0, 1, 3, 2, 4]
    cmsgs = [list(w[j][1]) for j in nbrs]
    tmsgs = [list(w[j][2]) for j in nbrs]
    ag.resilient_consensus_critic_hidden(cmsgs)
    ag.resilient_consensus_TR_hidden(tmsgs)
    ora.resilient_consensus_critic_hidden(cmsgs)
    ora.resilient_consensus_TR_hidden(tmsgs)
    assert all(m[0] >= EIG_GAP and m[1] >= SCORE_GAP for m in ora.last_margins), ora.last_margins
    for k in range(6):
        close(ag.critic.get_weights()[k], ora.critic[k], rtol=1e-4, atol=1e-5)
        close(ag.TR.get_weights()[k], ora.TR[k], rtol=1e-4, atol=1e-5)
    cagg, tagg = ag.resilient_consensus_critic(s, cmsgs), ag.resilient_consensus_TR(sa, tmsgs)
    wc, wt = ora.resilient_consensus_critic(s, cmsgs), ora.resilient_consensus_TR(sa, tmsgs)
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
        want, _ = DO.aggregate(X, H_)
        assert DO.margins(X, H_)[0] >= EIG_GAP and DO.margins(X, H_)[1] >= SCORE_GAP
        close(ag._resilient_aggregation(v).numpy(), want.reshape(3, 11), rtol=0,
              atol=out_atol(np.abs(v[np.isfinite(v)]).max()))
    with pytest.raises(K.L.RcmarlError):
        ag.H = 7
        ag._resilient_aggregation(v)
