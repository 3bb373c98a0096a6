"""GPU parity of adaptive robust clipping (rcmarl_arc_clip, include/rcmarl.h) against the oracle (tests/arc_oracle.py):
the kernel at n_in 1 .. 16, P 1 .. 1421 and every H, with inputs at odd offsets and row strides wider than P; d_k
bitwise scclip's; slots of +-inf and 1e30; bitwise determinism across calls, job orders and launch splits; and the
refusals.  Whole update rounds through Trainer: C2 with agent 4 Byzantine and every cooperative agent clipping, alone
or with nnm, bucketing or momentum, under clip, trim, scclip, mkrum, dnc and mda against alie, ipm, gauss, minmax_uv
and mimic; a 16-agent team where agents that clip sit beside plain, mixing and momentum agents; a world-1 PeerComm;
train_RPBCAC; and the per-agent API.

The factors c must match the fp64 oracle's to 1e-5 relative (fp32 distances over up to 1421 coordinates and one fp32
division); the set of clipped slots must be the oracle's except where a distance lies within 1e-5 of tau, where fp32
may rank it either way (c is then within rounding of 1 on both sides).  Given the kernel's own c, every row must equal
the fp32 restatement bit for bit, with every output pre-filled with NaN so that a write outside a job's rows fails.
In the update rounds the multi-Krum, dnc, mda and nnm oracles follow the kernel's selection at the near ties ARC
creates: a clipped row lies exactly as far from x_0 as the row that set tau.  After whole update rounds
weights rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 against the fp64 oracle (as test_trainer_gpu.py)."""
import datetime
import itertools

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import arc_oracle as AO                                # noqa: E402
import bucket_oracle as BO                             # noqa: E402
import dissensus_mimic_oracle as DM                    # noqa: E402
import momentum_oracle as MO                           # noqa: E402
import nnm_oracle as NO                                # noqa: E402
import subset_oracle as SO                             # noqa: E402
import team_util as TU                                 # noqa: E402
import vector_oracle as VO                             # noqa: E402
import test_bucketing_gpu as TB                        # noqa: E402  (the 16-agent round helpers)
import test_nnm_gpu as NG                              # noqa: E402  (the C2 round helpers)
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels            # noqa: E402
from kernel_util import synth                          # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f32, f64 = np.float32, np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
PS = (1, 31, 33, 661, 1421)
N_ROWS, S = 24, 1427                                   # message rows and their stride (wider than every P)
TIE = 1e-5


@pytest.fixture(scope="module")
def K():
    return load_kernels()


class Launches:
    """Device buffers of a set of jobs (n_in, P, H, nodes), each job j with n_in dst rows at stride S and n_in weights,
    all at odd float offsets and pre-filled with NaN; the message stack starts at float 3 of its buffer."""

    def __init__(self, K, cases):
        self.K, self.cases = K, cases
        self.msgs_buf = torch.full((3 + N_ROWS * S,), NAN, device=K.dev)
        self.dst = torch.full((len(cases), 5 + 16 * S), NAN, device=K.dev)
        self.w = torch.full((len(cases), 1 + 16 + 2), NAN, device=K.dev)

    def job(self, j):
        n_in, P, H, nodes = self.cases[j]
        return self.K.ops.vector_job(self.dst[j, 5:], self.msgs_buf[3:], S, P, nodes, H, self.K.L.MIX_ARC,
                                     weights_out=self.w[j, 1:])

    def load(self, stack):
        self.msgs_buf[3:].copy_(torch.as_tensor(stack.reshape(-1)))

    def out(self, j):
        """(rows [n_in, P], c [n_in]) of job j, after checking that nothing outside them was written."""
        n_in, P, _, _ = self.cases[j]
        d = self.dst[j].cpu().numpy()
        w = self.w[j].cpu().numpy()
        D = np.stack([d[5 + k * S:5 + k * S + P] for k in range(n_in)])
        mask = np.ones(d.shape, bool)
        for k in range(n_in):
            mask[5 + k * S:5 + k * S + P] = False
        assert np.isnan(d[mask]).all() and np.isnan(w[1 + n_in:]).all() and np.isnan(w[0]), \
            f"job {self.cases[j][:3]} wrote past its rows"
        return D, w[1:1 + n_in]


def _cases(rs):
    out = []
    for n_in in range(1, 17):
        for H in range(n_in):
            for P in PS:
                nodes = [int(x) for x in rs.choice(N_ROWS, size=n_in, replace=n_in > N_ROWS)]
                if n_in >= 3 and (n_in + P + H) % 3 == 1:
                    nodes[-1] = nodes[1]                                    # a repeated in-node: its own slot
                out.append((n_in, P, H, nodes))
    return out


def _stack(rs):
    centre = rs.randn(S)
    return (centre + rs.randn(N_ROWS, S) * rs.uniform(0.05, 3.0, size=(N_ROWS, 1))).astype(f32)


def _check_job(rows, c, X, H, tag):
    """c against the fp64 oracle (the clipped set up to near ties), and the rows bitwise against the fp32 restatement
    given the kernel's c.  Returns the number of near ties met."""
    n = X.shape[0]
    want_c, tau = AO.factors(X, H)
    d = AO.distances(X)
    close(c, want_c, rtol=1e-5, atol=1e-6, err_msg=tag)
    assert c[0] == 1, tag
    ties = 0
    for k in range(1, n):
        if (c[k] < 1) != (want_c[k] < 1):
            assert abs(d[k] - tau) <= TIE * max(tau, 1e-30), f"{tag}: slot {k} d={d[k]} tau={tau}"
            ties += 1
    assert ((c < 1) & np.isfinite(d)).sum() <= AO.k_clip(H, n), tag          # at most k_clip finite rows change
    np.testing.assert_array_equal(rows, AO.rows(X, c), err_msg=tag)
    return ties


def test_arc_clip_against_the_oracle(K):
    """Every n_in 1 .. 16, every H and P 1 .. 1421 (680 jobs) in launches of 32."""
    rs = np.random.RandomState(9100)
    cases = _cases(rs)
    assert len(cases) == 136 * len(PS)
    B = Launches(K, cases)
    stack = _stack(rs)
    B.load(stack)
    for g in range(0, len(cases), 32):
        K.ops.arc_clip([B.job(j) for j in range(g, min(g + 32, len(cases)))])
    ties = 0
    for j, (n_in, P, H, nodes) in enumerate(cases):
        rows, c = B.out(j)
        ties += _check_job(rows, c, stack[nodes, :P], H, f"n_in={n_in} P={P} H={H} nodes={nodes}")
        if H == 0:
            np.testing.assert_array_equal(rows, stack[nodes, :P])
    print(f"near ties met: {ties}")


@pytest.mark.parametrize("n_in", [2, 4, 8, 16])
def test_distances_are_bitwise_scclips(K, n_in):
    """scclip at H' = k_clip clips at the same tau as ARC, so with n_in a power of two (its weights are c_k / n_in, an
    exact division) its c_k must equal ARC's bit for bit for every k >= 1: the same d_k, the same ranking and the same
    division, on every P and H."""
    rs = np.random.RandomState(9150 + n_in)
    stack = torch.as_tensor(_stack(rs)).to(K.dev)
    for P in PS:
        for H in range(n_in):
            kc = AO.k_clip(H, n_in)
            if kc >= n_in - 1:
                continue
            nodes = [int(x) for x in rs.choice(N_ROWS, size=n_in, replace=False)]
            dst = torch.empty(n_in, S, device=K.dev)
            c = torch.full((n_in,), NAN, device=K.dev)
            K.ops.arc_clip([K.ops.vector_job(dst, stack, S, P, nodes, H, K.L.MIX_ARC, weights_out=c)])
            agg = torch.empty(P, device=K.dev)
            w = torch.full((n_in,), NAN, device=K.dev)
            K.ops.vector_aggregate([K.ops.vector_job(agg, stack, S, P, nodes, kc, "scclip", weights_out=w)])
            got, sc = c.cpu().numpy(), w.cpu().numpy() * f32(n_in)
            np.testing.assert_array_equal(got[1:], sc[1:], err_msg=f"P={P} H={H}")


def test_poisoned_slots_become_the_own_row(K):
    """Slots of +inf, -inf and 1e30: c = 0 and the row is x_0 bit for bit; every row is finite; no other slot's row
    differs from the oracle's restatement."""
    rs = np.random.RandomState(9200)
    stack = _stack(rs)
    stack[17, ::3] = np.inf
    stack[18, 1::4] = -np.inf
    stack[19] = 1e30
    stack[15, 5] = 1e30
    cases = [(16, 1421, 3, list(range(4, 20))), (4, 761, 1, [0, 17, 18, 19]), (7, 33, 2, [1, 2, 17, 3, 18, 4, 19]),
             (5, 1421, 4, [15, 17, 18, 19, 0]), (4, 1, 1, [2, 17, 3, 4])]
    B = Launches(K, cases)
    B.load(stack)
    K.ops.arc_clip([B.job(j) for j in range(len(cases))])
    for j, (n_in, P, H, nodes) in enumerate(cases):
        rows, c = B.out(j)
        X = stack[nodes, :P]
        bad = [k for k in range(1, n_in) if not np.isfinite(AO.distances(X)[k])]
        assert bad and all(c[k] == 0 for k in bad), (j, bad, c)
        for k in bad:
            np.testing.assert_array_equal(rows[k], X[0])
        if np.isfinite(X[0]).all():
            assert np.isfinite(rows).all()
        _check_job(rows, c, X, H, f"job {j}")


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(9300)
    cases = _cases(rs)[::23][:30]
    B = Launches(K, cases)
    B.load(_stack(rs))

    def run(order_groups):
        B.dst.fill_(NAN)
        B.w.fill_(NAN)
        for g in order_groups:
            K.ops.arc_clip([B.job(j) for j in g])
        return torch.nan_to_num(B.dst, 7.0).clone(), torch.nan_to_num(B.w, 7.0).clone()
    every = list(range(len(cases)))
    first = run([every])
    for groups in ([every], [every[::-1]], [every[5:9], every[:5], every[9:]], [[j] for j in every]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(9400)
    P = 700
    stack = rs.randn(8, P).astype(f32)
    msgs = torch.as_tensor(stack).to(K.dev)
    dst = torch.full((2, 4, P), NAN, device=K.dev)
    w = torch.full((2, 16), NAN, device=K.dev)
    J, A = K.ops.vector_job, K.L.MIX_ARC
    good = J(dst[0, 0], msgs, P, P, [0, 1, 2, 3], 1, A, weights_out=w[0])
    d, wo = dst[1, 0], w[1]
    bad = [J(d, msgs, P, P, [0, 1, 2], 1, K.L.MIX_NNM, weights_out=wo),     # another rule
           J(d, msgs, P, P, [0, 1, 2], 1, K.L.MIX_MOMENTUM, weights_out=wo),
           J(d, msgs, P, P, [0, 1, 2], 3, A, weights_out=wo),                  # H outside [0, n_in)
           J(d, msgs, P, P, [0, 1, 2], -1, A, weights_out=wo),
           J(d, msgs, P, P, [], 0, A, weights_out=wo),
           J(d, msgs, P, P, list(range(8)) * 2 + [0], 1, A, weights_out=wo),  # 17 in-nodes
           J(d, msgs, P, P, [0, -1, 2], 1, A, weights_out=wo),
           J(d, msgs, P, 0, [0, 1, 2], 1, A, weights_out=wo),
           J(msgs[2], msgs, P, P, [0, 1, 2], 1, A, weights_out=wo),            # dst row 0 is an in-node row
           J(d, msgs, P, P, [0, 1, 7], 1, A, weights_out=msgs[7]),             # weights on an in-node row
           J(dst[0, 2], msgs, P, P, [4, 5, 6], 1, A, weights_out=wo),          # dst rows on the other job's
           J(d, msgs, P, P, [4, 5, 6], 1, A, weights_out=w[0, 2:]),            # weights on the other job's
           J(d, msgs, P, P, [4, 5, 6], 1, A, weights_out=dst[1, 2]),           # weights on its own dst row 2
           J(d, msgs, P - 1, P, [4, 5, 6], 1, A, weights_out=wo)]              # its own dst rows overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.arc_clip([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(w).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.arc_clip([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(w).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.arc_clip([good])
    assert torch.isfinite(dst[0]).all() and torch.isfinite(w[0, :4]).all() and torch.isnan(w[0, 4:]).all()
    assert torch.isnan(dst[1]).all()


# ---------------------------------------------------------------------------------------------------------- Trainer
ATTACKS = {"alie": 1.5, "ipm": 0.5, "gauss": 0.3, "minmax_uv": 1.0, "mimic": 1}
C2_RULES = ("clip", "trim", "scclip", "mkrum", "dnc", "mda")
PRE = ("alone", "nnm", "bucket", "momentum")


def _c2_cases():
    out, names = [], list(ATTACKS)
    for r, rule in enumerate(C2_RULES):
        for p, pre in enumerate(PRE):
            if rule == "mkrum" and pre == "bucket":       # 3 bucketed rows cannot take mkrum at H = 1 (n >= H + 3)
                continue
            out.append((rule, pre, names[(r + p) % len(names)]))
    return out


class MkrumAgent(VO.RPBCACOracleAgent):
    """The multi-Krum oracle agent, following the kernel's selection where the scores are not clear.  A clipped row
    lies at distance tau from x_0, exactly as far as the row that set tau, so clipping creates ties of D_0k in exact
    arithmetic, where the rounding of the distances decides the selection.  kernel_w[epoch] = [critic w, TR w] of the
    agent's vector job (4 aggregations per epoch: critic, TR hidden; critic, TR estimates)."""

    kernel_w = None

    def _aggregate(self, w, msgs):
        X = np.stack([VO.AT.pack(m, self.dtype) for m in msgs])
        n, m = X.shape[0], X.shape[0] - self.H
        sc = np.sort(VO.krum_scores(X, self.H))
        c = len(self.last_weights)
        if m < n and (sc[m] - sc[m - 1]) <= 1e-4 * max(sc[m], 1e-30) and self.kernel_w is not None:
            keep = self.kernel_w[c // 4][c % 2][:n] > 0
            self.last_weights.append(keep / keep.sum())
            return VO.AT.unpack(SO.mean_of(X, np.flatnonzero(keep)), w)
        return super()._aggregate(w, msgs)


class MdaAgent(SO.RPBCACOracleAgent):
    """The MDA oracle agent, also following the kernel's selection where a candidate's diameter pair is not defined.
    SO.margin does not count a candidate whose diameter is the same pair of rows as the best's, since the kernel
    computes both from the same number.  A clipped row lies at distance tau from x_0, exactly as far as the row that
    set tau, so a candidate holding both has two pairs at its diameter in exact arithmetic: which one is the larger,
    and so whether two candidates share their diameter pair, is decided by rounding.  Where a candidate within 1e-6 of
    the best criterion has a second pair within 1e-6 of its diameter, the agent takes the kernel's selection."""

    def _aggregate(self, w, msgs):
        X = np.stack([SO.AT.pack(m, self.dtype) for m in msgs])
        c = len(self.last_weights)
        if self.kernel_w is not None and self._pair_ambiguous(X):
            keep = np.flatnonzero(self.kernel_w[c // 4][c % 2][:X.shape[0]] > 0)
            wt = np.zeros(X.shape[0], X.dtype)
            wt[keep] = 1.0 / len(keep)
            self.last_weights.append(wt)
            self.last_margins.append(0.0)
            return SO.AT.unpack(SO.mean_of(X, keep), w)
        return super()._aggregate(w, msgs)

    def _pair_ambiguous(self, X):
        s, cands = SO.candidates(X, self.H)
        if s < 3 or not cands:
            return False
        D = SO.distances(X)
        diam = [sorted((D[a, b] for a, b in itertools.combinations(S, 2)), reverse=True) for S in cands]
        best = min(d[0] for d in diam)
        return any(d[0] <= best * (1 + 1e-6) and d[0] - d[1] <= 1e-6 * d[0] for d in diam)


def _c2_agent(rule, w):
    if rule == "mda":
        return MdaAgent(w[0], w[1], w[2], 0.002, 0.01, 0.9, H=1, dtype=f64, aggregation=rule, gap=1e-4)
    if rule == "mkrum":
        return MkrumAgent(w[0], w[1], w[2], 0.002, 0.01, 0.9, H=1, dtype=f64, aggregation=rule)
    return NG._oracle_agent(rule, w, 0.01, 0.9, 1)


def _follow_mkrum(agents, runs):
    """Give each multi-Krum oracle agent the kernel's weights of epoch e from runs[e]."""
    for i, ag in enumerate(agents):
        if isinstance(ag, MkrumAgent):
            ag.kernel_w = [[tr.vec_weights[2 * tr.vec_agents.index(i) + t].cpu().numpy() for t in range(2)]
                           for tr in runs]


@pytest.mark.parametrize("rule,pre,kind", _c2_cases())
def test_c2_update_round_with_a_byzantine_agent(K, rule, pre, kind):
    """The benchmark's 5-agent team with agent 4 Byzantine and every cooperative agent clipping (H = 1, k_clip = 1)
    before `rule`, alone, with nnm, with bucketing (s = 2) or after momentum (beta 0.9): one update round of two epochs
    against the oracle with the hooks in the trainer's order (attack -> momentum -> ARC -> mixing); one ARC launch per
    epoch more than the same run without clipping, n_in = 4 clipped rows per agent, and the last epoch's factors."""
    w, desired, _ = pretrained()
    gamma, T, round_, N = 0.9, 40, 150, 64
    rs = np.random.RandomState(9500 + C2_RULES.index(rule))
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    mixing = {"nnm": "nnm", "bucket": ("bucket", 2)}.get(pre)
    momentum = 0.9 if pre == "momentum" else None
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule,
               momentum=momentum)
    tr, got, kernel_M, runs = NG._kernel_M(dict(cfg, clipping="arc"), rows, round_, mixing)
    assert tr.arc_agents == [0, 1, 2, 3]
    agents = [_c2_agent(rule, w[i]) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    NG._follow_dnc(agents, runs)
    SO.follow_kernel(agents, runs)
    _follow_mkrum(agents, runs)
    if kind == "mimic":
        inner = DM.StateHook(C2_BYZ, IN_NODES, {4: attack}, ["clip"] * 5, [1] * 5, seed=9, round_=round_, gap=1e-4)
        inner.follow = {e: r.mimic_targets() for e, r in enumerate(runs)}
    else:
        inner = AA.make_hook(C2_BYZ, IN_NODES, {4: attack}, seed=9, round_=round_)
    if momentum is not None:
        inner = MO.MomentumHook(agents, C2_BYZ, IN_NODES, [momentum] * 4 + [None], inner=inner)
    log = {}
    hook = AO.ArcHook(C2_BYZ, IN_NODES, ["arc"] * 4 + [None], [1] * 5, inner=inner, log=log)
    if pre == "nnm":
        hook = NO.mixing_hook(C2_BYZ, IN_NODES, ["nnm"] * 4 + [None], [1] * 5, inner=hook, kernel_M=kernel_M)
    elif pre == "bucket":
        hook = BO.bucketing_hook(C2_BYZ, IN_NODES, [mixing] * 4 + [None], 9, round_, inner=hook)
    want = AO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T, common_reward=False,
                           perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    factors = tr.clipping_factors()
    assert sorted(factors) == [0, 1, 2, 3]
    for i, c in factors.items():
        assert c.shape == (2, 4) and (c[:, 0] == 1).all() and ((c < 1).sum(1) <= 1).all()
        for t in range(2):
            close(c[t], log[i][-1][t][1], rtol=1e-2, atol=1e-3, err_msg=f"agent {i} net {t}")
    if rule in ("scclip", "mkrum", "dnc", "mda"):
        nw = tr.neighbour_weights()
        assert sorted(nw) == [0, 1, 2, 3] and all(v.shape == (2, 4) for v in nw.values())
        for v in nw.values():
            np.testing.assert_allclose(v.sum(1), 1.0, atol=1e-5)
    plain, _ = NG._trainer_round(cfg, rows, round_, 2, mixing)
    assert tr.launches - plain.launches == 2                                    # one ARC launch per epoch
    assert tr.msg_c.shape[0] - plain.msg_c.shape[0] == 4 * 4


def test_neighbour_weights_compose_through_the_factors(K):
    """For a whole-message rule w_eff_k = w'_k c_k (k >= 1) and w_eff_0 = w'_0 + sum w'_k (1 - c_k), with w' the
    rule's weights of the clipped rows (after any mixing matrix)."""
    w, desired, _ = pretrained()
    rs = np.random.RandomState(9600)
    rows = synth(rs, 40 * 16)
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=16, gamma=0.9, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=("ipm", 3.0),
               aggregation=["scclip", "mkrum", "dnc", "mda", "clip"], clipping="arc")
    for mixing in (None, [None, "nnm", None, ("bucket", 2), None]):
        tr, _ = NG._trainer_round(cfg, rows, 150, 2, mixing)
        nw, c, mats = tr.neighbour_weights(), tr.clipping_factors(), tr.mixing_matrices()
        for q, i in enumerate(tr.vec_agents + tr.dnc_agents + tr.subset_agents):
            src = (tr.vec_weights if i in tr.vec_agents else tr.dnc_weights if i in tr.dnc_agents
                   else tr.subset_weights)
            agents = tr.vec_agents if i in tr.vec_agents else tr.dnc_agents if i in tr.dnc_agents else tr.subset_agents
            r = agents.index(i)
            raw = src[2 * r:2 * r + 2, :len(tr._rule_nodes(i))].cpu().numpy().astype(f64)
            wp = np.einsum("tk,tkl->tl", raw, mats[i]) if i in mats else raw
            ci = c[i].astype(f64)
            want = wp * ci
            want[:, 0] = wp[:, 0] + (wp[:, 1:] * (1 - ci[:, 1:])).sum(1)
            close(nw[i], want.astype(f32), rtol=1e-6, atol=1e-7, err_msg=f"agent {i} mixing {mixing}")
            np.testing.assert_allclose(nw[i].sum(1), 1.0, atol=1e-5)


RULES16 = ["dnc", "clip", "gmed", "trim", "mkrum", "wmsr", "scclip", "krum"]   # the 8 cooperative agents, in order
MIX16 = [("bucket", 2), "nnm", None, None, ("bucket", 2), None, ("bucket", 3), None]
MOM16 = [None, None, 0.9, None, None, 0.99, None, None]
ARC16 = ["arc", "arc", "arc", "arc", None, "arc", None, None]


def test_16_agent_team_with_clipping_beside_plain_mixing_and_momentum_agents(K):
    """16 agents (8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy; in-neighbourhoods of 8): agents that clip alone,
    before nnm or bucketing and after momentum, beside agents that only bucket and one that does none of these."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mixing, mom, clip = ["clip"] * 16, [None] * 16, [None] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mixing[i], mom[i], clip[i] = RULES16[q], MIX16[q], MOM16[q], ARC16[q]
    H = [max(h, 1) if rules[i] == "dnc" or clip[i] else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[attacks.get(i) for i in range(16)], momentum=mom, clipping=clip)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    NG._follow_dnc(agents, runs)
    inner = AA.make_hook(labels, in_nodes, attacks, seed=4, round_=round_)
    inner = AO.ArcHook(labels, in_nodes, clip, H, inner=MO.MomentumHook(agents, labels, in_nodes, mom, inner=inner))
    want, _ = TB._oracle_round(agents, labels, in_nodes, rows, inner, mixing, H, N, T, round_, seed=4,
                               kernel_M=kernel_M)
    assert tr.arc_agents == [coop[q] for q in (0, 1, 2, 3, 5)] and len(tr.mom_agents) == 2
    assert tr._momentum_nodes(coop[2]) == list(range(tr.mom_row[coop[2]], tr.mom_row[coop[2]] + 8))
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(),
                   msg=f"agent {i} ({labels[i]}, {rules[i]}, {mixing[i]}, {mom[i]}, {clip[i]})")


def _round_cfg():
    w, desired, _ = pretrained()
    return dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1, fast_lr=0.01,
                slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                aggregation=["dnc", "scclip", "trim", "clip", "clip"], momentum=[0.9, None, None, None, None],
                mixing=[None, None, None, "nnm", None], clipping=["arc", "arc", None, "arc", None], attack=("mimic", 3))


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


def test_world1_peer_comm_with_clipping_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents clip."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    runs = []
    for bound in (False, True):
        tr = Trainer(**_round_cfg())
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append(NG._state(tr) + [tr.arc_weights.clone()])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_train_rpbcac_with_clipping_agents(K):
    """Drop-in path: train_RPBCAC with RPBCAC_agent objects that clip runs the same rounds as a Trainer built from the
    same objects with the same clipping passed directly, bit for bit, with one launch per epoch more than a run
    without clipping, and different weights."""
    import contextlib
    import io
    from rcmarl import api
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)
    clip = ["arc", None, "arc", "arc", None]

    def objects(with_clipping):
        env, agents, args = api.build_reference_objects(cfg)
        if with_clipping:
            for i in range(4):
                agents[i].clipping = clip[i]
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    env, agents, args = objects(True)
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(env, agents, args)
    tr = training.train_RPBCAC.last_trainer
    assert tr.clipping == clip and tr.arc_agents == [0, 2, 3]
    env2, agents2, args2 = objects(False)
    direct = training.build_trainer(env2, agents2, args2, clipping=clip)
    plain = training.build_trainer(*objects(False))
    for t in (direct, plain):
        for _ in range(2):
            t.rollout_block(4)
            t.update_round()
    torch.cuda.synchronize()
    assert direct.launches == tr.launches == plain.launches + 2 * 2            # one ARC launch per epoch
    for i in range(5):
        for a, b in zip(tr.get_weights(i), direct.get_weights(i)):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
    assert any(not np.array_equal(x, y) for i in range(4) for a, b in zip(tr.get_weights(i), plain.get_weights(i))
               for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------- agent API
@pytest.mark.parametrize("rule,mixing,momentum", [("clip", None, None), ("scclip", None, None), ("scclip", None, 0.9)])
def test_rpbcac_agent_methods_with_clipping(K, rule, mixing, momentum):
    """RPBCAC_agent(..., clipping="arc"): three rounds of hidden consensus, estimate consensus and projection step
    against the oracle agent fed the oracle's clipped rows (after the momentum step), with one neighbour far off so
    that ARC clips it.  (ARC before nnm is checked through the trainer, where the oracle can follow the kernel's nnm
    selections: a clipped row is exactly as far from x_0 as the row that set tau, a tie the rounding decides.)"""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H = 1
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule,
                      mixing=mixing, momentum=momentum, clipping="arc")
    ora = NG._oracle_agent(rule, w[0], 0.01, 0.9, H)
    rs = np.random.RandomState(9700)
    M = [None, None]
    for round_ in range(3):
        nbrs = [0, 1, 3, 2, 4]
        scale = [0.05, 0.05, 0.05, 0.05, 2.0]
        cmsgs = [[np.asarray(x) + rs.randn(*np.shape(x)).astype(f32) * sc for x in w[j][1]] for j, sc in zip(nbrs, scale)]
        tmsgs = [[np.asarray(x) + rs.randn(*np.shape(x)).astype(f32) * sc for x in w[j][2]] for j, sc in zip(nbrs, scale)]
        per = []
        for net, (msgs, mine) in enumerate(((cmsgs, ora.critic), (tmsgs, ora.TR))):
            X = np.stack([MO.AT.pack(m, f64) for m in msgs])
            if momentum is not None:
                X, M[net] = MO.step(X, MO.AT.pack(mine, f64), M[net], momentum, round_ == 0)
            Y, c, _ = AO.clip(X, H)
            assert c[-1] < 1
            per.append([MO.AT.unpack(Y[k], msgs[0]) for k in range(Y.shape[0])])
        ag.resilient_consensus_critic_hidden(cmsgs)
        ag.resilient_consensus_TR_hidden(tmsgs)
        ora.resilient_consensus_critic_hidden(per[0])
        ora.resilient_consensus_TR_hidden(per[1])
        cagg, tagg = ag.resilient_consensus_critic(s, cmsgs), ag.resilient_consensus_TR(sa, tmsgs)
        wc, wt = ora.resilient_consensus_critic(s, per[0]), ora.resilient_consensus_TR(sa, per[1])
        close(cagg.numpy(), wc, rtol=1e-4, atol=1e-5)
        close(tagg.numpy(), wt, rtol=1e-4, atol=1e-5)
        ag.critic_update_team(s, cagg)
        ag.TR_update_team(sa, tagg)
        ora.critic_update_team(s, wc)
        ora.TR_update_team(sa, wt)
        for k in range(6):
            close(ag.critic.get_weights()[k], ora.critic[k], rtol=1e-4, atol=1e-5)
            close(ag.TR.get_weights()[k], ora.TR[k], rtol=1e-4, atol=1e-5)
