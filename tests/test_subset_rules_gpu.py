"""GPU parity of the exact subset-selection rules MDA and SMEA (rcmarl_subset_aggregate, include/rcmarl.h) against the
float64 oracle (tests/subset_oracle.py): the kernel at n_in 1, 2, 3, 4, 7 and 16 over every allowed H, P 1 .. 1421,
repeated in-nodes and 32 jobs per launch; bitwise identities with DnC, multi-Krum and the own row; exact ties; Byzantine
rows of 1e30 / +-inf; bitwise determinism; the staging bound in a fresh process and the refusals; whole update rounds
through Trainer with a Byzantine agent, a 16-agent team mixing mda / smea with the other rules under nnm and
bucketing, a world-1 PeerComm, and the per-agent API.

Selections are compared exactly where the oracle's margin is clear: a relative gap between the best and second-best
criterion of at least 1e-9 for MDA (fp64 distances from the same fp32 inputs, summed in another order) and 1e-6 for
SMEA (Jacobi in the kernel, LAPACK here); there dst must equal the oracle's fp32 mean bit for bit.  Elsewhere dst must
be the bitwise mean of the rows the kernel selected, and their criterion must lie within 1e-8 (MDA) or 1e-5 (SMEA) of
the oracle's minimum, relative.  In whole update rounds the oracle agents follow the kernel's selection below a margin
of 1e-4; weights rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as test_dnc_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import subset_oracle as SO                             # noqa: E402
import team_util as TU                                 # noqa: E402
import test_bucketing_gpu as BG                        # noqa: E402  (the mixed-round helpers)
import test_nnm_gpu as NG                              # noqa: E402  (the C2 round helpers)
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
C2_BYZ = ["Cooperative"] * 4 + ["Byzantine"]
ATTACKS = {"alie": 1.5, "ipm": 0.5, "gauss": 0.3, "minmax_uv": 1.0}
PS = (1, 661, 761, 1101, 1421)
GAP = {"mda": 1e-9, "smea": 1e-6}
SLACK = {"mda": 1e-8, "smea": 1e-5}
# In whole update rounds the oracle's fp64 messages drift from the kernel's fp32 ones by about 1e-6, relative, so there
# the oracle follows the kernel's selection below a margin of 1e-4 (the min-max attacks place their message at the
# honest diameter, where MDA's candidates nearly tie).
ROUND_GAP = 1e-4


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def rule_id(K, rule):
    return K.L.SUBSET_RULES[rule]


def subset_job(K, dst, msgs, P, nodes, H, rule, weights_out=None):
    return K.ops.vector_job(dst, msgs, msgs.shape[1], P, nodes, H, rule_id(K, rule), weights_out=weights_out)


def _stack(rs, n_rows=24, P=max(PS)):
    """Messages around a common centre (as trained networks are), each row with its own spread."""
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def check_job(rule, X32, H, got, gw, tag):
    """One job's dst [P] and weights [n_in] against the oracle; True if the selection was compared exactly."""
    n_in = X32.shape[0]
    X = X32.astype(f64)
    kept = gw > 0
    s = n_in - max(H, int(SO.flagged(X).sum()))
    assert kept.sum() == s, (tag, gw)
    assert (gw[kept] == np.float32(1) / np.float32(s)).all(), tag
    assert (gw[~kept] == 0).all(), tag
    sel = tuple(np.flatnonzero(kept))
    np.testing.assert_array_equal(got, SO.mean_of(X32, sel), err_msg=tag)     # the fp32 mean, bit for bit
    want = SO.select(rule, X, H)
    if SO.margin(rule, X, H) >= GAP[rule]:
        assert sel == want, (tag, sel, want)
        return True
    D = SO.distances(X)
    c_got, c_min = SO.criterion(rule, D, sel), SO.criterion(rule, D, want)
    assert c_got - c_min <= SLACK[rule] * max(abs(c_min), 1e-30), (tag, c_got, c_min)
    return False


# ---------------------------------------------------------------------------------------------------------- kernel
def _cases():
    """(rule, n_in, H, P, repeated) over n_in in {1, 2, 3, 4, 7, 16}, every allowed H, both rules."""
    out = []
    for rule in SO.RULES:
        for n_in in (1, 2, 3, 4, 7, 16):
            for H in range(n_in):
                out.append((rule, n_in, H, PS[(n_in + H) % 5], (n_in + H) % 3 == 1 and n_in >= 3))
    return out


def _jobs(K, rs, msgs, stack, cases, dst, wout):
    jobs, spec = [], []
    for j, (rule, n_in, H, P, rep) in enumerate(cases):
        nodes = [int(x) for x in rs.choice(stack.shape[0], size=n_in, replace=False)]
        if rep:
            nodes[-1] = nodes[int(rs.randint(0, n_in - 1))]                     # a repeated in-node
        jobs.append(subset_job(K, dst[j], msgs, P, nodes, H, rule, weights_out=wout[j]))
        spec.append((rule, n_in, H, P, rep, nodes))
    return jobs, spec


def test_subset_aggregate_against_the_oracle(K):
    """Both rules at n_in 1, 2, 3, 4, 7, 16, every H, P 1 .. 1421, repeated in-nodes, launches of 32 jobs: weights_out
    and dst against the fp64 oracle, selections exactly where the margin is clear."""
    rs = np.random.RandomState(5100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases()
    n_exact = 0
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
        wout = torch.full((len(part), 16), NAN, device=K.dev)
        jobs, spec = _jobs(K, rs, msgs, stack, part, dst, wout)
        K.ops.subset_aggregate(jobs)
        got, gw = dst.cpu().numpy(), wout.cpu().numpy()
        for j, (rule, n_in, H, P, rep, nodes) in enumerate(spec):
            tag = f"{rule} n_in={n_in} H={H} P={P} nodes={nodes}"
            assert np.isnan(got[j, P:]).all() and np.isnan(gw[j, n_in:]).all(), f"{tag}: wrote past n / n_in"
            n_exact += check_job(rule, stack[nodes, :P], H, got[j, :P], gw[j, :n_in], tag)
    print(f"subset jobs {len(cases)}, selections compared exactly {n_exact}")
    assert n_exact >= 0.8 * len(cases), n_exact


def test_identities_with_dnc_mkrum_and_the_own_row(K):
    """H = 0 gives DnC's output at H = 0 bit for bit, and multi-Krum's where n_in >= 3; H = n - 1 gives x_0."""
    rs = np.random.RandomState(5200)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    P = stack.shape[1]
    for n_in in (1, 2, 3, 4, 7, 16):
        nodes = [int(x) for x in rs.choice(24, size=n_in, replace=False)]
        ref = torch.full((2, P), NAN, device=K.dev)
        K.ops.dnc_aggregate([K.ops.vector_job(ref[0], msgs, P, P, nodes, 0, K.L.SPECTRAL_DNC)])
        if n_in >= 3:
            K.ops.vector_aggregate([K.ops.vector_job(ref[1], msgs, P, P, nodes, 0, "mkrum")])
        for rule in SO.RULES:
            d = torch.full((2, P), NAN, device=K.dev)
            w = torch.full((2, 16), NAN, device=K.dev)
            K.ops.subset_aggregate([subset_job(K, d[0], msgs, P, nodes, 0, rule, weights_out=w[0]),
                                    subset_job(K, d[1], msgs, P, nodes, n_in - 1, rule, weights_out=w[1])])
            assert torch.equal(d[0], ref[0]), (rule, n_in)
            if n_in >= 3:
                assert torch.equal(d[0], ref[1]), (rule, n_in)
            np.testing.assert_array_equal(d[1].cpu().numpy(), stack[nodes[0]])
            np.testing.assert_array_equal(w[1, :n_in].cpu().numpy(), np.eye(n_in)[0])
            np.testing.assert_array_equal(w[0, :n_in].cpu().numpy(), np.full(n_in, np.float32(1) / np.float32(n_in)))


def test_exact_ties_select_the_lowest_rank(K):
    """Repeated rows: in-nodes (a, a, b, b) at H = 2 tie {0, 1} and {2, 3} at 0 under both rules; (p, q, p, q) at H = 1
    ties every MDA candidate at D_pq; every row equal ties every candidate at 0."""
    rs = np.random.RandomState(5300)
    stack = _stack(rs, n_rows=6, P=761)
    stack[5] = stack[4]
    msgs = to_dev(K, stack)[0]
    P = 761
    cases = [(rule, [1, 1, 2, 2], 2, (0, 1)) for rule in SO.RULES]
    cases += [(rule, [2, 2, 1, 1], 2, (0, 1)) for rule in SO.RULES]
    cases += [("mda", [0, 3, 0, 3], 1, (0, 1, 2))]
    cases += [(rule, [4] * 7 + [5] * 5, H, tuple(range(12 - H))) for rule in SO.RULES for H in (0, 3, 7, 11)]
    dst = torch.full((len(cases), P), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    K.ops.subset_aggregate([subset_job(K, dst[j], msgs, P, nodes, H, rule, weights_out=wout[j])
                            for j, (rule, nodes, H, _) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (rule, nodes, H, want) in enumerate(cases):
        assert tuple(np.flatnonzero(gw[j, :len(nodes)] > 0)) == want, (rule, nodes, H, gw[j])
        assert SO.select(rule, stack[nodes].astype(f64), H) == want
        np.testing.assert_array_equal(got[j], SO.mean_of(stack[nodes], want))


def test_byzantine_rows_get_weight_zero(K):
    """Rows holding +-inf (whole, or in some coordinates) and rows of +-1e30, at most H of them: weight 0, a finite
    aggregate equal to the oracle's; every row flagged gives the own row."""
    rs = np.random.RandomState(5400)
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
                         (16, 7, [16, 17, 18]), (3, 1, [19]), (12, 5, [17]), (7, 3, [16, 19])]:
        honest = [int(x) for x in rs.choice(np.arange(1, 16), size=n_in - 1 - len(bad), replace=False)]
        nodes = [0] + [int(x) for x in rs.permutation(honest + bad)]                  # own (row 0) is honest
        for rule in SO.RULES:
            cases.append((rule, n_in, H, nodes))
    dst = torch.full((len(cases), P), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    K.ops.subset_aggregate([subset_job(K, dst[j], msgs, P, nodes, H, rule, weights_out=wout[j])
                            for j, (rule, n_in, H, nodes) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (rule, n_in, H, nodes) in enumerate(cases):
        is_bad = np.array([k in huge or k in infs for k in nodes])
        assert np.isfinite(got[j]).all(), nodes
        assert (gw[j, :n_in][is_bad] == 0).all(), (rule, nodes, gw[j, :n_in])
        check_job(rule, stack[nodes], H, got[j], gw[j, :n_in], f"{rule} {nodes} H={H}")
    for rule in SO.RULES:
        d, w = torch.full((P,), NAN, device=K.dev), torch.full((16,), NAN, device=K.dev)
        K.ops.subset_aggregate([subset_job(K, d, msgs, P, [17, 18, 17], 1, rule, weights_out=w)])
        np.testing.assert_array_equal(d.cpu().numpy(), stack[17])
        np.testing.assert_array_equal(w.cpu().numpy()[:3], [1, 0, 0])


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(5500)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases()[::2][:32]
    dst = torch.full((len(cases), stack.shape[1]), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    jobs, _ = _jobs(K, rs, msgs, stack, cases, dst, wout)
    assert len(jobs) == 32 and {c[1] for c in cases} >= {1, 4, 16} and {c[0] for c in cases} == {"mda", "smea"}

    def run(groups):
        dst.fill_(NAN)
        wout.fill_(NAN)
        for g in groups:
            K.ops.subset_aggregate(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(wout, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_dst_and_weights_untouched(K):
    rs = np.random.RandomState(5600)
    stack = _stack(rs, n_rows=8, P=700)
    msgs = to_dev(K, stack)[0]
    P = 700
    dst = torch.full((3, P), NAN, device=K.dev)
    wout = torch.full((3, 16), NAN, device=K.dev)
    V = K.ops.vector_job
    M = K.L.SUBSET_SMEA
    good = V(dst[0], msgs, P, P, [0, 1, 2, 3], 1, M, weights_out=wout[0])
    d, w = dst[1], wout[1]
    bad = [V(d, msgs, P, P, [0, 1, 2], 3, M, weights_out=w),                    # H >= n_in
           V(d, msgs, P, P, [0, 1, 2], -1, M, weights_out=w),
           V(d, msgs, P, P, [], 0, M, weights_out=w),
           V(d, msgs, P, P, list(range(8)) * 2 + [0], 0, M, weights_out=w),     # 17 in-nodes
           V(d, msgs, P, P, [0, -1, 2], 0, M, weights_out=w),
           V(d, msgs, P, P, [0, 1, 2], 0, 2, weights_out=w),                    # not a subset rule
           V(d, msgs, P, P, [0, 1, 2], 0, -1, weights_out=w),
           V(d, msgs, P, 0, [0, 1, 2], 0, M, weights_out=w),
           V(msgs[2], msgs, P, P, [0, 1, 2], 0, M, weights_out=w),              # dst is an in-node row
           V(msgs[3][3:], msgs, P, P, [5, 6, 7], 0, M, weights_out=w),          # dst overlaps a row of the other job
           V(d, msgs, P, 48 * 1024 // 3 + 1, [0, 1, 2], 0, M, weights_out=w),   # over the staging bound
           V(d, msgs, P, P, [0, 1, 2], 0, M, weights_out=msgs[1][5:]),          # weights_out on an in-node row
           V(d, msgs, P, P, [0, 1, 2], 0, M, weights_out=dst[0][10:]),          # ... on the other job's dst
           V(d, msgs, P, P, [0, 1, 2], 0, M, weights_out=wout[0][3:]),          # ... on its weights_out
           V(dst[0][1:], msgs, P, P - 1, [0, 1, 2], 0, M, weights_out=w)]       # two dsts overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.subset_aggregate([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(wout).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.subset_aggregate([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(wout).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.subset_aggregate([good])
    assert torch.isfinite(dst[0]).all() and torch.isnan(dst[1:]).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import subset_oracle as SO
rs = np.random.RandomState(5700)
for rule, n_in, P, H in (("smea", 16, 3072, 3), ("mda", 4, 3072, 1), ("mda", 16, 3072, 2)):
    X = (rs.randn(n_in, P) * rs.uniform(0.1, 1, size=(n_in, 1)) + rs.randn(P)).astype(np.float32)
    msgs = torch.as_tensor(X).cuda()
    dst = torch.full((P,), float("nan"), device="cuda")
    w = torch.full((n_in,), float("nan"), device="cuda")
    ops.subset_aggregate([ops.vector_job(dst, msgs, P, P, list(range(n_in)), H, L.SUBSET_RULES[rule], weights_out=w)])
    sel = tuple(np.flatnonzero(w.cpu().numpy() > 0))
    assert len(sel) == n_in - H, sel
    assert np.array_equal(dst.cpu().numpy(), SO.mean_of(X, sel)), (rule, n_in)
    Xd = X.astype(np.float64)
    assert SO.margin(rule, Xd, H) < 1e-6 or sel == SO.select(rule, Xd, H), (rule, sel)
print("ok")
"""


def test_staging_bound_as_the_first_launch_of_a_process(K, tmp_path):
    """Static shared memory counts against the default 48 KB too: a job at RCMARL_SUBSET_MAX_FLOATS (n_in 16 x 3072)
    runs as the first launch of a fresh process, then jobs of 48 KB of dynamic staging."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    assert 16 * 3072 == K.L.SUBSET_MAX_FLOATS and 4 * 3072 == 12288
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
def _subset_agent(rule, w, fast, gamma, H):
    return SO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, aggregation=rule,
                                gap=ROUND_GAP)


def _check_neighbour_weights(tr, agents):
    """neighbour_weights of the subset agents against the oracle's last-epoch weights (times M for agents that mix)."""
    got = tr.neighbour_weights()
    mats = tr.mixing_matrices()
    for i in tr.subset_agents:
        want = np.stack(agents[i].last_weights[-4:-2]).astype(f64)    # the last epoch's critic and TR aggregations
        if i in mats:
            want = np.einsum("tk,tkl->tl", want, mats[i].astype(f64))
        assert got[i].shape == (2, len(tr.in_nodes[i]))
        close(got[i], want, rtol=1e-6, atol=1e-7, err_msg=f"agent {i}")


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("kind", list(ATTACKS))
@pytest.mark.parametrize("rule", SO.RULES)
def test_c2_update_round_with_a_byzantine_agent(K, rule, kind, N):
    """The benchmark's 5-agent team with agent 4 Byzantine, every cooperative agent on `rule` (H = 1): one update
    round of two epochs against the oracle's round with the per-receiver hook; one subset launch per epoch more than on
    clip, and one aggregate row per cooperative agent."""
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(5800 + N)
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack)
    tr, got, _, runs = NG._kernel_M(dict(cfg, aggregation=rule), rows, round_, None)
    agents = [_subset_agent(rule, w[i], 0.01, gamma, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    SO.follow_kernel(agents, runs)
    hook = AA.make_hook(C2_BYZ, IN_NODES, {4: attack}, seed=9, round_=round_)
    want = SO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                           common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    assert tr.subset_agents == [0, 1, 2, 3] and tr.msg_c.shape[0] == 5 + 3 + 4
    _check_neighbour_weights(tr, agents)
    plain, _ = NG._trainer_round(dict(cfg, aggregation="clip"), rows, round_, 2, None)
    assert tr.launches - plain.launches == 2                                    # one subset launch per epoch
    assert plain.neighbour_weights() == {} and plain.msg_c.shape[0] == 5 + 3


RULES16 = ["mda", "clip", "smea", "trim", "mkrum", "dnc", "smea", "mda"]   # the 8 cooperative agents, in order
MIX16 = [("bucket", 2), "nnm", None, ("bucket", 2), ("bucket", 2), "nnm", ("bucket", 3), None]


def test_16_agent_team_mixing_subset_rules_with_the_others_under_nnm_and_bucketing(K):
    """16 agents (8 cooperative, 5 Byzantine with mixed attacks, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, receiver
    0 listing Byzantine agent 1 twice) with the cooperative agents' rules and mixing set per agent: mda and smea beside
    coordinate-wise, distance-based and dnc rules, with and without nnm or bucketing."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mixing = ["clip"] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mixing[i] = RULES16[q], MIX16[q]
    H = [max(h, 1) if rules[i] in ("dnc", "mda", "smea") else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(_subset_agent(rules[i], w[i], fast[i], gamma, H[i]) if rules[i] in SO.RULES
                          else NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[attacks.get(i) for i in range(16)])
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    NG._follow_dnc(agents, runs)
    SO.follow_kernel(agents, runs)
    inner = AA.make_hook(labels, in_nodes, attacks, seed=4, round_=round_)
    want, log = BG._oracle_round(agents, labels, in_nodes, rows, inner, mixing, H, N, T, round_, seed=4,
                                 kernel_M=kernel_M)
    assert tr.subset_agents == [i for i in coop if rules[i] in SO.RULES] and len(tr.subset_agents) == 4
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]}, {mixing[i]})")
    _check_neighbour_weights(tr, agents)


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


def test_world1_peer_comm_with_subset_rules_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents use mda and smea."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["mda", "mkrum", "smea", "dnc", "clip"], attack=("minmax_std", 1.0),
                     mixing=[None, None, "nnm", None, None])
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append([getattr(tr, n).clone() for n in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v",
                                                      "vec_weights", "dnc_weights", "subset_weights")])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


# ---------------------------------------------------------------------------------------------------------- agent API
@pytest.mark.parametrize("rule", SO.RULES)
def test_rpbcac_agent_methods_with_subset_rules(K, rule):
    """RPBCAC_agent(..., aggregation="mda" | "smea"): hidden consensus, estimate consensus, projection step and
    _resilient_aggregation against the oracle agent."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H = 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule)
    ora = _subset_agent(rule, w[0], 0.01, 0.9, H)
    nbrs = [0, 1, 3, 2, 4]
    cmsgs = [list(w[j][1]) for j in nbrs]
    tmsgs = [list(w[j][2]) for j in nbrs]
    ag.resilient_consensus_critic_hidden(cmsgs)
    ag.resilient_consensus_TR_hidden(tmsgs)
    ora.resilient_consensus_critic_hidden(cmsgs)
    ora.resilient_consensus_TR_hidden(tmsgs)
    assert all(m >= ROUND_GAP for m in ora.last_margins), ora.last_margins
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
        X = v.reshape(7, -1)
        want, _ = SO.aggregate(rule, X, H_)                      # fp32: the kernel's output bit for bit
        assert SO.margin(rule, X.astype(f64), H_) >= GAP[rule]
        np.testing.assert_array_equal(ag._resilient_aggregation(v).numpy(), want.reshape(3, 11))
    with pytest.raises(K.L.RcmarlError):
        ag.H = 7
        ag._resilient_aggregation(v)
