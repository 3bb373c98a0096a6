"""GPU parity of the iterative outlier scissor (rcmarl_ios_aggregate, include/rcmarl.h) against the float64 oracle
(tests/ios_oracle.py): the kernel at n_in 1, 2, 3, 4, 7 and 16 over every H, P 1 .. 1421, repeated in-nodes and 32 jobs
per launch; bitwise identities with DnC, MDA and multi-Krum at H = 0; exact ties; Byzantine rows of 1e30 / +-inf;
bitwise determinism; the staging bound in a fresh process and the refusals; whole update rounds through Trainer with a
Byzantine agent under six receiver-agnostic attacks, a 16-agent team mixing ios with the other rules under nnm,
bucketing, momentum and ARC, a world-1 PeerComm, and the per-agent API.

Selections are compared exactly where the oracle's margin is clear: a relative gap between the largest and the next
distance of at least 1e-9 at every removal (fp64 centres and distances from the same fp32 inputs, summed in another
order); there dst must equal the oracle's fp32 mean bit for bit.  Elsewhere dst must be the bitwise mean of the rows
the kernel kept, and every row it removed must have been within 1e-9 of the largest distance, relative, when it went.
In whole update rounds the oracle agents follow the kernel's selection below a margin of 1e-4; weights rtol 1e-3 /
atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as test_subset_rules_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import arc_oracle as AO                                # noqa: E402
import dissensus_mimic_oracle as DM                    # noqa: E402
import ios_oracle as IO                                # noqa: E402
import momentum_oracle as MO                           # noqa: E402
import team_util as TU                                 # noqa: E402
import test_bucketing_gpu as BG                        # noqa: E402  (the mixed-round helpers)
import test_nnm_gpu as NG                              # noqa: E402  (the C2 round helpers)
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
ATTACKS = {"alie": 1.5, "ipm": 0.5, "gauss": 0.3, "minmax_std": 1.0, "dissensus": 1.0, "mimic": 1}
PS = (1, 661, 761, 1101, 1421)
GAP = 1e-9
# In whole update rounds the oracle's fp64 messages drift from the kernel's fp32 ones by about 1e-6, relative, so there
# the oracle follows the kernel's selection below a margin of 1e-4.
ROUND_GAP = 1e-4


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def ios_job(K, dst, msgs, P, nodes, H, weights_out=None):
    return K.ops.vector_job(dst, msgs, msgs.shape[1], P, nodes, H, K.L.FILTER_IOS, weights_out=weights_out)


def _stack(rs, n_rows=24, P=max(PS)):
    """Messages around a common centre (as trained networks are), each row with its own spread."""
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def check_job(X32, H, got, gw, tag):
    """One job's dst [P] and weights [n_in] against the oracle; True if the selection was compared exactly."""
    n_in = X32.shape[0]
    X = X32.astype(f64)
    kept = gw > 0
    s = n_in - max(H, int(IO.flagged(X).sum()))
    assert kept.sum() == s, (tag, gw)
    assert (gw[kept] == np.float32(1) / np.float32(s)).all(), tag
    assert (gw[~kept] == 0).all(), tag
    sel = tuple(np.flatnonzero(kept))
    np.testing.assert_array_equal(got, IO.mean_of(X32, sel), err_msg=tag)     # the fp32 mean, bit for bit
    if IO.margin(X, H) >= GAP:
        assert sel == IO.kept(X, H), (tag, sel, IO.kept(X, H))
        return True
    U = [k for k in range(n_in) if not IO.flagged(X)[k]]                        # replay the kernel's removals
    while len(U) > s:
        d = IO.distances(X, U)
        top = max(d.values())
        gone = [k for k in U if k not in sel and d[k] >= top * (1 - GAP)]
        assert gone, (tag, sel, d)
        U.remove(max(gone, key=lambda k: (d[k], k)))
    assert tuple(U) == sel, (tag, U, sel)
    return False


# ---------------------------------------------------------------------------------------------------------- kernel
def _cases():
    """(n_in, H, P, repeated) over n_in in {1, 2, 3, 4, 7, 16} and every allowed H."""
    out = []
    for n_in in (1, 2, 3, 4, 7, 16):
        for H in range(n_in):
            out.append((n_in, H, PS[(n_in + H) % 5], (n_in + H) % 3 == 1 and n_in >= 3))
    return out


def _jobs(K, rs, msgs, stack, cases, dst, wout):
    jobs, spec = [], []
    for j, (n_in, H, P, rep) in enumerate(cases):
        nodes = [int(x) for x in rs.choice(stack.shape[0], size=n_in, replace=False)]
        if rep:
            nodes[-1] = nodes[int(rs.randint(0, n_in - 1))]                     # a repeated in-node
        jobs.append(ios_job(K, dst[j], msgs, P, nodes, H, weights_out=wout[j]))
        spec.append((n_in, H, P, rep, nodes))
    return jobs, spec


def test_ios_aggregate_against_the_oracle(K):
    """n_in 1, 2, 3, 4, 7, 16, every H, P 1 .. 1421, repeated in-nodes, launches of up to 32 jobs: weights_out and dst
    against the fp64 oracle, selections exactly where the margin is clear."""
    rs = np.random.RandomState(6100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases() * 2
    n_exact = 0
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
        wout = torch.full((len(part), 16), NAN, device=K.dev)
        jobs, spec = _jobs(K, rs, msgs, stack, part, dst, wout)
        K.ops.ios_aggregate(jobs)
        got, gw = dst.cpu().numpy(), wout.cpu().numpy()
        for j, (n_in, H, P, rep, nodes) in enumerate(spec):
            tag = f"n_in={n_in} H={H} P={P} nodes={nodes}"
            assert np.isnan(got[j, P:]).all() and np.isnan(gw[j, n_in:]).all(), f"{tag}: wrote past n / n_in"
            n_exact += check_job(stack[nodes, :P], H, got[j, :P], gw[j, :n_in], tag)
    print(f"ios jobs {len(cases)}, selections compared exactly {n_exact}")
    assert n_exact >= 0.8 * len(cases), n_exact


def test_identities_with_dnc_mda_and_mkrum_at_H0(K):
    """H = 0 gives the plain mean: DnC's and MDA's outputs at H = 0 bit for bit, and multi-Krum's where n_in >= 3."""
    rs = np.random.RandomState(6200)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    P = stack.shape[1]
    for n_in in (1, 2, 3, 4, 7, 16):
        nodes = [int(x) for x in rs.choice(24, size=n_in, replace=False)]
        ref = torch.full((3, P), NAN, device=K.dev)
        K.ops.dnc_aggregate([K.ops.vector_job(ref[0], msgs, P, P, nodes, 0, K.L.SPECTRAL_DNC)])
        K.ops.subset_aggregate([K.ops.vector_job(ref[1], msgs, P, P, nodes, 0, K.L.SUBSET_MDA)])
        if n_in >= 3:
            K.ops.vector_aggregate([K.ops.vector_job(ref[2], msgs, P, P, nodes, 0, "mkrum")])
        d = torch.full((P,), NAN, device=K.dev)
        w = torch.full((16,), NAN, device=K.dev)
        K.ops.ios_aggregate([ios_job(K, d, msgs, P, nodes, 0, weights_out=w)])
        assert torch.equal(d, ref[0]) and torch.equal(d, ref[1]), n_in
        if n_in >= 3:
            assert torch.equal(d, ref[2]), n_in
        np.testing.assert_array_equal(w[:n_in].cpu().numpy(), np.full(n_in, np.float32(1) / np.float32(n_in)))
        np.testing.assert_array_equal(d.cpu().numpy(), IO.mean_of(stack[nodes], range(n_in)))


def test_exact_ties_remove_the_higher_index_first(K):
    """Rows v, -v, s v, -s v (s a sign per coordinate) are all at the same distance from their mean 0: H = 1 removes
    row 3.  In-nodes (a, a, b, b) tie at H = 1 and remove row 3; two rows left tie and keep the lower; every row equal
    ties at 0 and keeps the first n - H."""
    rs = np.random.RandomState(6300)
    P = 761
    stack = _stack(rs, n_rows=10, P=P)
    v = stack[6].copy()
    sgn = np.where(rs.rand(P) < 0.5, -1, 1).astype(np.float32)
    stack[6], stack[7], stack[8], stack[9] = v, -v, sgn * v, -sgn * v
    stack[5] = stack[4]
    msgs = to_dev(K, stack)[0]
    cases = [([6, 7, 8, 9], 1, (0, 1, 2)), ([9, 8, 7, 6], 1, (0, 1, 2)), ([1, 1, 2, 2], 1, (0, 1, 2)),
             ([2, 2, 1, 1], 1, (0, 1, 2)), ([1, 2], 1, (0,)), ([3, 0], 1, (0,)), ([0, 3, 1], 2, None)]
    cases += [([4] * 7 + [5] * 5, H, tuple(range(12 - H))) for H in (0, 3, 7, 11)]
    dst = torch.full((len(cases), P), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    K.ops.ios_aggregate([ios_job(K, dst[j], msgs, P, nodes, H, weights_out=wout[j])
                         for j, (nodes, H, _) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (nodes, H, want) in enumerate(cases):
        sel = tuple(np.flatnonzero(gw[j, :len(nodes)] > 0))
        want = want or IO.kept(stack[nodes].astype(f64), H)
        assert sel == want, (nodes, H, gw[j])
        assert IO.kept(stack[nodes].astype(f64), H) == want
        np.testing.assert_array_equal(got[j], IO.mean_of(stack[nodes], want))


def test_byzantine_rows_get_weight_zero(K):
    """Rows holding +-inf (whole, or in some coordinates) and rows of +-1e30, at most H of them: weight 0, a finite
    aggregate equal to the oracle's; every row flagged gives the own row."""
    rs = np.random.RandomState(6400)
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
        cases.append((n_in, H, [0] + [int(x) for x in rs.permutation(honest + bad)]))   # own (row 0) is honest
    dst = torch.full((len(cases), P), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    K.ops.ios_aggregate([ios_job(K, dst[j], msgs, P, nodes, H, weights_out=wout[j])
                         for j, (n_in, H, nodes) in enumerate(cases)])
    got, gw = dst.cpu().numpy(), wout.cpu().numpy()
    for j, (n_in, H, nodes) in enumerate(cases):
        is_bad = np.array([k in huge or k in infs for k in nodes])
        assert np.isfinite(got[j]).all(), nodes
        assert (gw[j, :n_in][is_bad] == 0).all(), (nodes, gw[j, :n_in])
        check_job(stack[nodes], H, got[j], gw[j, :n_in], f"{nodes} H={H}")
    d, w = torch.full((P,), NAN, device=K.dev), torch.full((16,), NAN, device=K.dev)
    K.ops.ios_aggregate([ios_job(K, d, msgs, P, [17, 18, 17], 1, weights_out=w)])
    np.testing.assert_array_equal(d.cpu().numpy(), stack[17])
    np.testing.assert_array_equal(w.cpu().numpy()[:3], [1, 0, 0])


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(6500)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = (_cases() * 2)[::2][:32]
    dst = torch.full((len(cases), stack.shape[1]), NAN, device=K.dev)
    wout = torch.full((len(cases), 16), NAN, device=K.dev)
    jobs, _ = _jobs(K, rs, msgs, stack, cases, dst, wout)
    assert len(jobs) == 32 and {c[0] for c in cases} >= {1, 4, 16}

    def run(groups):
        dst.fill_(NAN)
        wout.fill_(NAN)
        for g in groups:
            K.ops.ios_aggregate(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(wout, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_dst_and_weights_untouched(K):
    rs = np.random.RandomState(6600)
    stack = _stack(rs, n_rows=8, P=700)
    msgs = to_dev(K, stack)[0]
    P = 700
    dst = torch.full((3, P), NAN, device=K.dev)
    wout = torch.full((3, 16), NAN, device=K.dev)
    V = K.ops.vector_job
    M = K.L.FILTER_IOS
    good = V(dst[0], msgs, P, P, [0, 1, 2, 3], 1, M, weights_out=wout[0])
    d, w = dst[1], wout[1]
    bad = [V(d, msgs, P, P, [0, 1, 2], 3, M, weights_out=w),                    # H >= n_in
           V(d, msgs, P, P, [0, 1, 2], -1, M, weights_out=w),
           V(d, msgs, P, P, [], 0, M, weights_out=w),
           V(d, msgs, P, P, list(range(8)) * 2 + [0], 0, M, weights_out=w),     # 17 in-nodes
           V(d, msgs, P, P, [0, -1, 2], 0, M, weights_out=w),
           V(d, msgs, P, P, [0, 1, 2], 0, 1, weights_out=w),                    # not an ios rule
           V(d, msgs, P, P, [0, 1, 2], 0, -1, weights_out=w),
           V(d, msgs, P, 0, [0, 1, 2], 0, M, weights_out=w),
           V(msgs[2], msgs, P, P, [0, 1, 2], 0, M, weights_out=w),              # dst is an in-node row
           V(msgs[3][3:], msgs, P, P, [5, 6, 7], 0, M, weights_out=w),          # dst overlaps a row of the other job
           V(d, msgs, P, 48 * 1024 // 5 + 1, [0, 1, 2], 0, M, weights_out=w),   # over the staging bound
           V(d, msgs, P, P, [0, 1, 2], 0, M, weights_out=msgs[1][5:]),          # weights_out on an in-node row
           V(d, msgs, P, P, [0, 1, 2], 0, M, weights_out=dst[0][10:]),          # ... on the other job's dst
           V(d, msgs, P, P, [0, 1, 2], 0, M, weights_out=wout[0][3:]),          # ... on its weights_out
           V(dst[0][1:], msgs, P, P - 1, [0, 1, 2], 0, M, weights_out=w)]       # two dsts overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.ios_aggregate([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(wout).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.ios_aggregate([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(wout).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.ios_aggregate([good])
    assert torch.isfinite(dst[0]).all() and torch.isnan(dst[1:]).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import ios_oracle as IO
rs = np.random.RandomState(6700)
for n_in, P, H in ((16, 2730, 3), (4, 8192, 1), (16, 2730, 15)):
    X = (rs.randn(n_in, P) * rs.uniform(0.1, 1, size=(n_in, 1)) + rs.randn(P)).astype(np.float32)
    msgs = torch.as_tensor(X).cuda()
    dst = torch.full((P,), float("nan"), device="cuda")
    w = torch.full((n_in,), float("nan"), device="cuda")
    ops.ios_aggregate([ops.vector_job(dst, msgs, P, P, list(range(n_in)), H, L.FILTER_IOS, weights_out=w)])
    sel = tuple(np.flatnonzero(w.cpu().numpy() > 0))
    assert len(sel) == n_in - H, sel
    assert np.array_equal(dst.cpu().numpy(), IO.mean_of(X, sel)), (n_in, H)
    Xd = X.astype(np.float64)
    assert IO.margin(Xd, H) < 1e-9 or sel == IO.kept(Xd, H), (n_in, H, sel)
print("ok")
"""


def test_staging_bound_as_the_first_launch_of_a_process(K, tmp_path):
    """Static shared memory counts against the default 48 KB too: jobs at RCMARL_IOS_MAX_FLOATS ((16 + 2) x 2730 and
    (4 + 2) x 8192 floats) run as the first launches of a fresh process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    assert 18 * 2730 <= K.L.IOS_MAX_FLOATS < 18 * 2731 and 6 * 8192 == K.L.IOS_MAX_FLOATS
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
def _ios_agent(w, fast, gamma, H):
    return IO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, gap=ROUND_GAP)


def _check_neighbour_weights(tr, agents):
    """neighbour_weights of the ios agents against the oracle's last-epoch weights (times M for agents that mix)."""
    got = tr.neighbour_weights()
    mats = tr.mixing_matrices()
    for i in tr.ios_agents:
        want = np.stack(agents[i].last_weights[-4:-2]).astype(f64)    # the last epoch's critic and TR aggregations
        if i in mats:
            want = np.einsum("tk,tkl->tl", want, mats[i].astype(f64))
        assert got[i].shape == (2, len(tr.in_nodes[i]))
        close(got[i], want, rtol=1e-6, atol=1e-7, err_msg=f"agent {i}")


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("kind", list(ATTACKS))
def test_c2_update_round_with_a_byzantine_agent(K, kind, N):
    """The benchmark's 5-agent team with agent 4 Byzantine, every cooperative agent on ios (H = 1): one update round
    of two epochs against the oracle's round with the per-receiver hook; one ios launch per epoch more than on clip,
    and one aggregate row per cooperative agent."""
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(6800 + N)
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack)
    tr, got, _, runs = NG._kernel_M(dict(cfg, aggregation="ios"), rows, round_, None)
    agents = [_ios_agent(w[i], 0.01, gamma, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    IO.follow_kernel(agents, runs)
    if kind in ("dissensus", "mimic"):
        hook = DM.StateHook(C2_BYZ, IN_NODES, {4: attack}, ["clip"] * 5, [1] * 5, seed=9, round_=round_, gap=1e-4)
        hook.follow = {e: r.mimic_targets() for e, r in enumerate(runs)}
    else:
        hook = AA.make_hook(C2_BYZ, IN_NODES, {4: attack}, seed=9, round_=round_)
    want = IO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                           common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    assert tr.ios_agents == [0, 1, 2, 3] and tr.msg_c.shape[0] == 5 + 3 + 4
    _check_neighbour_weights(tr, agents)
    plain, _ = NG._trainer_round(dict(cfg, aggregation="clip"), rows, round_, 2, None)
    assert tr.launches - plain.launches == 2                                    # one ios launch per epoch
    assert plain.neighbour_weights() == {} and plain.msg_c.shape[0] == 5 + 3


RULES16 = ["ios", "clip", "ios", "trim", "mkrum", "dnc", "ios", "ios"]   # the 8 cooperative agents, in order
MIX16 = [("bucket", 2), "nnm", None, None, ("bucket", 2), None, ("bucket", 3), "nnm"]
MOM16 = [None, None, 0.9, None, None, 0.99, None, None]
ARC16 = ["arc", "arc", "arc", "arc", None, "arc", None, None]


def test_16_agent_team_mixing_ios_with_the_others_under_nnm_bucketing_momentum_and_arc(K):
    """16 agents (8 cooperative, 5 Byzantine with mixed attacks, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, receiver
    0 listing Byzantine agent 1 twice): ios agents that bucket and clip, keep momentum and clip, bucket, and mix by nnm,
    beside coordinate-wise, distance-based and dnc agents with their own pre-aggregation steps."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mixing, mom, clip = ["clip"] * 16, [None] * 16, [None] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mixing[i], mom[i], clip[i] = RULES16[q], MIX16[q], MOM16[q], ARC16[q]
    H = [max(h, 1) if rules[i] in ("dnc", "ios") or clip[i] else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(_ios_agent(w[i], fast[i], gamma, H[i]) if rules[i] == "ios"
                          else NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[attacks.get(i) for i in range(16)], momentum=mom, clipping=clip)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    NG._follow_dnc(agents, runs)
    IO.follow_kernel(agents, runs)
    inner = AA.make_hook(labels, in_nodes, attacks, seed=4, round_=round_)
    inner = AO.ArcHook(labels, in_nodes, clip, H, inner=MO.MomentumHook(agents, labels, in_nodes, mom, inner=inner))
    want, _ = BG._oracle_round(agents, labels, in_nodes, rows, inner, mixing, H, N, T, round_, seed=4,
                               kernel_M=kernel_M)
    assert tr.ios_agents == [coop[q] for q in (0, 2, 6, 7)]
    assert tr._rule_nodes(coop[2]) == list(range(tr.arc_row[coop[2]], tr.arc_row[coop[2]] + 8))
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(),
                   msg=f"agent {i} ({labels[i]}, {rules[i]}, {mixing[i]}, {mom[i]}, {clip[i]})")
    nw = tr.neighbour_weights()
    for i in tr.ios_agents:
        assert nw[i].shape == (2, 8)
        np.testing.assert_allclose(nw[i].sum(1), 1.0, atol=1e-5)


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


def test_world1_peer_comm_with_ios_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents use ios."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["ios", "mkrum", "ios", "dnc", "clip"], attack=("minmax_std", 1.0),
                     mixing=[None, None, "nnm", None, None], clipping=["arc", None, None, None, None])
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append([getattr(tr, n).clone() for n in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v",
                                                      "vec_weights", "dnc_weights", "ios_weights", "msg_c", "msg_t")])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


# ---------------------------------------------------------------------------------------------------------- agent API
def test_rpbcac_agent_methods_with_ios(K):
    """RPBCAC_agent(..., aggregation="ios"): hidden consensus, estimate consensus, projection step and
    _resilient_aggregation against the oracle agent."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H = 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation="ios")
    ora = _ios_agent(w[0], 0.01, 0.9, H)
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
        want, _ = IO.aggregate(X, H_)                            # fp32: the kernel's output bit for bit
        assert IO.margin(X.astype(f64), H_) >= GAP
        np.testing.assert_array_equal(ag._resilient_aggregation(v).numpy(), want.reshape(3, 11))
    with pytest.raises(K.L.RcmarlError):
        ag.H = 7
        ag._resilient_aggregation(v)
