"""GPU parity of per-neighbour momentum (rcmarl_momentum_mix, include/rcmarl.h) against the oracle
(tests/momentum_oracle.py): the kernel over 5 consecutive steps carrying its state at n_in 1, 2, 3, 4, 7, 16, P 1, 31,
32, 33, 1421 and beta 0, 0.5, 0.9, with inputs at odd offsets and rows strides wider than P; slots of +-inf and 1e30;
bitwise determinism across calls, job orders and launch splits; and the refusals.  Whole update rounds through
Trainer: C2 with agent 4 Byzantine and every cooperative agent on momentum under clip, scclip, dnc and mda against alie,
minmax_uv and mimic; a 16-agent team where momentum agents sit beside plain agents and agents that mix; a checkpoint
between two rounds; a world-1 PeerComm; train_RPBCAC; and the per-agent API.

M and the momentum rows must equal the fp32 oracle's bit for bit (every operation is rounded on its own on both sides),
with every output pre-filled with NaN so that a write outside a job's rows fails.  After whole update rounds weights
rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 against the fp64 oracle (as test_trainer_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import dissensus_mimic_oracle as DM                    # noqa: E402
import momentum_oracle as MO                           # noqa: E402
import subset_oracle as SO                             # noqa: E402
import team_util as TU                                 # noqa: E402
import test_bucketing_gpu as TB                        # noqa: E402  (the 16-agent round helpers)
import test_nnm_gpu as NG                              # noqa: E402  (the C2 round helpers)
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, synth     # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f32, f64 = np.float32, np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
N_INS = (1, 2, 3, 4, 7, 16)
PS = (1, 31, 32, 33, 1421)
BETAS = (0.0, 0.5, 0.9)
N_ROWS, S = 24, 1427                                   # message rows and their stride (wider than every P)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


class Launches:
    """Device buffers of a set of jobs, each job j with n_in dst rows at stride S, n_in M rows at stride MS = P + 13
    and a ref, all at odd float offsets, pre-filled with NaN; the message stack starts at float 3 of its buffer."""

    def __init__(self, K, cases):
        self.K, self.cases = K, cases
        self.msgs_buf = torch.full((3 + N_ROWS * S,), NAN, device=K.dev)
        self.dst = torch.full((len(cases), 5 + 16 * S), NAN, device=K.dev)
        self.M = torch.full((len(cases), 7 + 16 * (1421 + 13)), NAN, device=K.dev)
        self.ref = torch.full((len(cases), 1 + 1421 + 2), NAN, device=K.dev)

    def job(self, j, first):
        n_in, P, beta, nodes = self.cases[j]
        return self.K.ops.momentum_job(self.dst[j, 5:], self.msgs_buf[3:], S, P, nodes, self.ref[j, 1:], self.M[j, 7:],
                                       P + 13, beta, first)

    def load(self, stack, refs):
        """stack [N_ROWS, S] float32 messages; refs [n_jobs, 1421] float32."""
        self.msgs_buf[3:].copy_(torch.as_tensor(stack.reshape(-1)))
        for j, (_, P, _, _) in enumerate(self.cases):
            self.ref[j, 1:1 + P].copy_(torch.as_tensor(refs[j, :P]))

    def rows(self, j):
        """(dst rows [n_in, P], M rows [n_in, P]) of job j, after checking that nothing outside them was written."""
        n_in, P, _, _ = self.cases[j]
        d = self.dst[j].cpu().numpy()
        m = self.M[j].cpu().numpy()
        D = np.stack([d[5 + k * S:5 + k * S + P] for k in range(n_in)])
        Mr = np.stack([m[7 + k * (P + 13):7 + k * (P + 13) + P] for k in range(n_in)])
        dmask = np.ones(d.shape, bool)
        mmask = np.ones(m.shape, bool)
        for k in range(n_in):
            dmask[5 + k * S:5 + k * S + P] = False
            mmask[7 + k * (P + 13):7 + k * (P + 13) + P] = False
        assert np.isnan(d[dmask]).all() and np.isnan(m[mmask]).all(), f"job {self.cases[j][:3]} wrote past its rows"
        return D, Mr


def _cases(rs):
    out = []
    for n_in in N_INS:
        for P in PS:
            for beta in BETAS:
                nodes = [int(x) for x in rs.choice(N_ROWS, size=n_in, replace=False)]
                if n_in >= 3 and (n_in + P) % 2 == 1:
                    nodes[-1] = nodes[0]                                    # a repeated in-node: its own slot
                out.append((n_in, P, beta, nodes))
    return out


def _stack(rs):
    centre = rs.randn(S)
    return (centre + rs.randn(N_ROWS, S) * rs.uniform(0.05, 2.0, size=(N_ROWS, 1))).astype(f32), centre


def test_momentum_mix_against_the_oracle_over_five_steps(K):
    """90 jobs in launches of 30, 5 steps with new messages and references each step: M and the rows bitwise."""
    rs = np.random.RandomState(8100)
    cases = _cases(rs)
    assert len(cases) == 90
    B = Launches(K, cases)
    state = [None] * len(cases)
    for step in range(5):
        stack, centre = _stack(rs)
        refs = (centre[:1421] + rs.randn(len(cases), 1421) * 0.3).astype(f32)
        B.load(stack, refs)
        for g in range(0, len(cases), 30):
            K.ops.momentum_mix([B.job(j, step == 0) for j in range(g, min(g + 30, len(cases)))])
        for j, (n_in, P, beta, nodes) in enumerate(cases):
            rows, M = B.rows(j)
            want_rows, state[j] = MO.step(stack[nodes, :P], refs[j, :P], state[j], beta, step == 0)
            tag = f"step {step} n_in={n_in} P={P} beta={beta} nodes={nodes}"
            np.testing.assert_array_equal(M, state[j], err_msg=tag)
            np.testing.assert_array_equal(rows, want_rows, err_msg=tag)
            if beta == 0.0:
                close(rows, stack[nodes, :P], rtol=2 ** -22, atol=1e-6, err_msg=tag)


def test_poisoned_slots_stay_in_their_rows(K):
    """Slots of +inf, -inf and 1e30 (from step 1 on, then gone at step 3): every row and M bitwise as the oracle's; a
    +-inf coordinate stays +-inf in its slot's M and row for good, and no other slot's row is touched."""
    rs = np.random.RandomState(8200)
    cases = [(16, 1421, 0.9, list(range(16))), (4, 761, 0.5, [0, 17, 18, 19]), (7, 33, 0.0, [1, 2, 17, 3, 18, 4, 19])]
    B = Launches(K, cases)
    state = [None] * 3
    for step in range(5):
        stack, centre = _stack(rs)
        if step in (1, 2):
            stack[17, ::3] = np.inf
            stack[18, 1::4] = -np.inf
            stack[19] = 1e30
            stack[15, :5] = np.inf
        refs = (centre[:1421] + rs.randn(3, 1421) * 0.3).astype(f32)
        B.load(stack, refs)
        K.ops.momentum_mix([B.job(j, step == 0) for j in range(3)])
        for j, (n_in, P, beta, nodes) in enumerate(cases):
            rows, M = B.rows(j)
            want, state[j] = MO.step(stack[nodes, :P], refs[j, :P], state[j], beta, step == 0)
            np.testing.assert_array_equal(M, state[j], err_msg=f"step {step} job {j}")
            np.testing.assert_array_equal(rows, want, err_msg=f"step {step} job {j}")
            bad = [k for k, r in enumerate(nodes) if r in (15, 17, 18)]
            if step >= 1:
                for k in bad:
                    assert not np.isfinite(M[k]).all()
                good = [k for k in range(n_in) if k not in bad and nodes[k] != 19]
                assert np.isfinite(rows[good]).all() and np.isfinite(M[good]).all()
    rows, M = B.rows(1)
    assert (M[1, ::3] == np.inf).all() and (rows[1, ::3] == np.inf).all()           # sticky after 2 clean steps
    assert (M[2, 1::4] == -np.inf).all() and (rows[2, 1::4] == -np.inf).all()
    assert np.isfinite(M[3]).all() and np.abs(rows[3]).max() > 1e20                 # 1e30 decays at beta 0.5, finite


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(8300)
    cases = _cases(rs)[::3][:30]
    B = Launches(K, cases)
    stack, centre = _stack(rs)
    B.load(stack, (centre[:1421] + rs.randn(len(cases), 1421) * 0.3).astype(f32))
    M0 = (torch.randn(B.M.shape, device=K.dev) * 0.3)

    def run(order_groups):
        B.dst.fill_(NAN)
        B.M.copy_(M0)
        for g in order_groups:
            K.ops.momentum_mix([B.job(j, 0) for j in g])
        return torch.nan_to_num(B.dst, 7.0).clone(), B.M.clone()
    every = list(range(len(cases)))
    first = run([every])
    for groups in ([every], [every[::-1]], [every[5:9], every[:5], every[9:]], [[j] for j in every]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(8400)
    P = 700
    stack = rs.randn(8, P).astype(f32)
    msgs = torch.as_tensor(stack).to(K.dev)
    dst = torch.full((2, 4, P), NAN, device=K.dev)
    M = torch.full((2, 4, P), NAN, device=K.dev)
    ref = torch.full((2, P), NAN, device=K.dev)
    ref[:] = torch.as_tensor(stack[0])
    J = K.ops.momentum_job
    good = J(dst[0, 0], msgs, P, P, [0, 1, 2, 3], ref[0], M[0, 0], P, 0.9, 1)
    d, m, c = dst[1, 0], M[1, 0], ref[1]
    bad = [J(d, msgs, P, P, [0, 1, 2], c, m, P, 1.0, 1),                        # beta outside [0, 1)
           J(d, msgs, P, P, [0, 1, 2], c, m, P, -0.25, 1),
           J(d, msgs, P, P, [0, 1, 2], c, m, P, float("inf"), 1),
           J(d, msgs, P, P, [0, 1, 2], c, m, P, float("nan"), 1),
           J(d, msgs, P, P, [0, 1, 2], c, m, P, 0.5, 2),                        # first not 0 / 1
           J(d, msgs, P, P, [], c, m, P, 0.5, 1),
           J(d, msgs, P, P, list(range(8)) * 2 + [0], c, m, P, 0.5, 1),         # 17 in-nodes
           J(d, msgs, P, P, [0, -1, 2], c, m, P, 0.5, 1),
           J(d, msgs, P, 0, [0, 1, 2], c, m, P, 0.5, 1),
           J(msgs[2], msgs, P, P, [0, 1, 2], c, m, P, 0.5, 1),                  # dst row 0 is an in-node row
           J(d, msgs, P, P, [0, 1, 7], c, msgs[5], P, 0.5, 1),                  # M row 2 is in-node row 7
           J(d, msgs, P, P, [0, 1, 2], msgs[1], m, P, 0.5, 1),                  # ref is an in-node row
           J(d, msgs, P, P, [0, 1, 2], dst[0, 1], m, P, 0.5, 1),                # ref on the other job's dst row 1
           J(dst[0, 2], msgs, P, P, [4, 5, 6], c, m, P, 0.5, 1),                # dst rows on the other job's
           J(d, msgs, P, P, [4, 5, 6], c, M[0, 3], P, 0.5, 1),                  # M rows on the other job's M row 3
           J(d, msgs, P, P, [4, 5, 6], c, dst[1, 1], P, 0.5, 1),                # M rows on its own dst rows
           J(d, msgs, P, P, [4, 5, 6], c, m, P - 1, 0.5, 1),                    # its own M rows overlap
           J(d, msgs, P, P, [4, 5, 6], M[0, 1], m, P, 0.5, 1)]                  # ref on the other job's M row 1
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.momentum_mix([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(M).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.momentum_mix([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(M).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.momentum_mix([good])
    assert torch.isfinite(dst[0]).all() and torch.isfinite(M[0]).all() and torch.isnan(dst[1]).all()


# ---------------------------------------------------------------------------------------------------------- Trainer
C2_ATTACKS = {"alie": 1.5, "minmax_uv": 1.0, "mimic": 1}


def _c2_agent(rule, w):
    if rule == "mda":
        return SO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, 0.01, 0.9, H=1, dtype=f64, aggregation=rule, gap=1e-4)
    return NG._oracle_agent(rule, w, 0.01, 0.9, 1)


@pytest.mark.parametrize("kind", list(C2_ATTACKS))
@pytest.mark.parametrize("rule", ["clip", "scclip", "dnc", "mda"])
def test_c2_update_round_with_a_byzantine_agent(K, rule, kind):
    """The benchmark's 5-agent team with agent 4 Byzantine and every cooperative agent on momentum (beta 0.9) before
    `rule` (H = 1): one update round of two epochs against the oracle with the momentum hook around the attack hook;
    one momentum launch per epoch more than without momentum, and n_in = 4 momentum rows per agent."""
    w, desired, _ = pretrained()
    gamma, T, round_, N = 0.9, 40, 150, 64
    rs = np.random.RandomState(8500)
    rows = synth(rs, T * N)
    attack = (kind, C2_ATTACKS[kind])
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule)
    tr, got, _, runs = NG._kernel_M(dict(cfg, momentum=0.9), rows, round_, None)
    assert tr.mom_agents == [0, 1, 2, 3] and tr.momentum_steps == [2] * 4
    agents = [_c2_agent(rule, w[i]) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    NG._follow_dnc(agents, runs)
    SO.follow_kernel(agents, runs)
    if kind == "mimic":
        inner = DM.StateHook(C2_BYZ, IN_NODES, {4: attack}, ["clip"] * 5, [1] * 5, seed=9, round_=round_, gap=1e-4)
        inner.follow = {e: r.mimic_targets() for e, r in enumerate(runs)}
    else:
        inner = AA.make_hook(C2_BYZ, IN_NODES, {4: attack}, seed=9, round_=round_)
    hook = MO.MomentumHook(agents, C2_BYZ, IN_NODES, [0.9] * 4 + [None], inner=inner)
    want = MO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T, common_reward=False,
                           perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    for q, i in enumerate(tr.mom_agents):                    # the carried state itself
        for t in range(2):
            P = tr.PC if t == 0 else tr.PT
            got_M = tr.momentum_M[q, t, :4, :P].cpu().numpy()
            close(got_M, hook.M[(i, t)], rtol=1e-3, atol=5e-5, err_msg=f"agent {i} net {t}")
    if rule in ("scclip", "dnc", "mda"):
        nw = tr.neighbour_weights()
        assert sorted(nw) == [0, 1, 2, 3] and all(v.shape == (2, 4) for v in nw.values())
        for v in nw.values():
            np.testing.assert_allclose(v.sum(1), 1.0, atol=1e-5)
    plain, _ = NG._trainer_round(cfg, rows, round_, 2, None)
    assert tr.launches - plain.launches == 2                                    # one momentum launch per epoch
    assert tr.msg_c.shape[0] - plain.msg_c.shape[0] == 4 * 4


RULES16 = ["dnc", "clip", "gmed", "trim", "mkrum", "wmsr", "scclip", "krum"]   # the 8 cooperative agents, in order
MIX16 = [("bucket", 2), "nnm", None, None, ("bucket", 2), None, ("bucket", 3), None]
MOM16 = [None, None, 0.9, 0.5, None, 0.99, None, None]


def test_16_agent_team_with_momentum_beside_plain_and_mixing_agents(K):
    """16 agents (8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy; in-neighbourhoods of 8): three cooperative agents
    on momentum (n_in = 8 rows each) beside agents that mix by nnm or bucketing and one that does neither."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mixing, mom = ["clip"] * 16, [None] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mixing[i], mom[i] = RULES16[q], MIX16[q], MOM16[q]
    H = [max(h, 1) if rules[i] == "dnc" else h for i, h in enumerate(H)]
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
               aggregation=rules, attack=[attacks.get(i) for i in range(16)], momentum=mom)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    NG._follow_dnc(agents, runs)
    inner = MO.MomentumHook(agents, labels, in_nodes, mom, inner=AA.make_hook(labels, in_nodes, attacks, seed=4,
                                                                              round_=round_))
    want, _ = TB._oracle_round(agents, labels, in_nodes, rows, inner, mixing, H, N, T, round_, seed=4,
                               kernel_M=kernel_M)
    assert tr.mom_agents == [coop[2], coop[3], coop[5]] and len(tr.mix_agents) == 4
    assert tr.msg_c.shape[0] == 16 + len(tr.byz_pairs) + 4 + 1 + (5 + 8 + 5 + 4) + 3 * 8
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(),
                   msg=f"agent {i} ({labels[i]}, {rules[i]}, {mixing[i]}, {mom[i]})")


def _round_cfg():
    w, desired, _ = pretrained()
    return dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1, fast_lr=0.01,
                slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                aggregation=["dnc", "scclip", "trim", "clip", "clip"], momentum=[0.9, 0.99, 0.5, None, None],
                mixing=[None, None, None, "nnm", None], attack=("mimic", 3))


def test_checkpoint_between_rounds_is_bitwise(K, tmp_path):
    """Round 1, save, load into a fresh trainer, round 2: bitwise the two rounds run straight through, momentum state
    and step counts included.  A checkpoint without the momentum state, or of another shape, is refused."""
    from rcmarl.trainer import Trainer
    straight = Trainer(**_round_cfg())
    for _ in range(2):
        straight.rollout_block()
        straight.update_round()
    first = Trainer(**_round_cfg())
    first.rollout_block()
    first.update_round()
    first.save(tmp_path / "ck.pt")
    sd = first.state_dict()
    assert sd["momentum_steps"] == [2, 2, 2] and tuple(sd["momentum_M"].shape) == (3, 2, 16, first.PT)
    resumed = Trainer(**_round_cfg())
    resumed.load(tmp_path / "ck.pt")
    resumed.rollout_block()
    resumed.update_round()
    torch.cuda.synchronize()
    assert resumed.momentum_steps == straight.momentum_steps == [4, 4, 4]
    for a, b in zip(NG._state(resumed) + [resumed.momentum_M], NG._state(straight) + [straight.momentum_M]):
        assert torch.equal(a, b)
    fresh = Trainer(**_round_cfg())
    for drop in ("momentum_M", "momentum_steps"):
        with pytest.raises(K.L.RcmarlError, match="momentum"):
            fresh.load_state_dict({k: v for k, v in sd.items() if k != drop})
    with pytest.raises(K.L.RcmarlError, match="momentum"):
        fresh.load_state_dict(dict(sd, momentum_M=sd["momentum_M"][:2]))
    with pytest.raises(K.L.RcmarlError, match="momentum"):
        Trainer(**dict(_round_cfg(), momentum=[0.9, None, None, None, None])).load_state_dict(sd)
    plain = Trainer(**dict(_round_cfg(), momentum=None))
    assert "momentum_M" not in plain.state_dict()
    plain.load_state_dict(sd)                                     # a trainer without momentum ignores the state


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


def test_world1_peer_comm_with_momentum_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents keep momentum."""
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
        runs.append(NG._state(tr) + [tr.momentum_M.clone()])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_train_rpbcac_with_momentum_agents(K):
    """Drop-in path: train_RPBCAC with RPBCAC_agent objects that keep momentum runs the same rounds as a Trainer built
    from the same objects with the same momentum passed directly, bit for bit, with one launch per epoch more than a
    run without momentum, and different weights."""
    import contextlib
    import io
    from rcmarl import api
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)
    mom = [0.9, None, 0.5, 0.99, None]

    def objects(with_momentum):
        env, agents, args = api.build_reference_objects(cfg)
        if with_momentum:
            for i in range(4):
                agents[i].momentum = mom[i]
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    env, agents, args = objects(True)
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(env, agents, args)
    tr = training.train_RPBCAC.last_trainer
    assert tr.momentum == mom and tr.mom_agents == [0, 2, 3]
    env2, agents2, args2 = objects(False)
    direct = training.build_trainer(env2, agents2, args2, momentum=mom)
    plain = training.build_trainer(*objects(False))
    for t in (direct, plain):
        for _ in range(2):
            t.rollout_block(4)
            t.update_round()
    torch.cuda.synchronize()
    assert direct.launches == tr.launches == plain.launches + 2 * 2            # one momentum launch per epoch
    for i in range(5):
        for a, b in zip(tr.get_weights(i), direct.get_weights(i)):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
    assert any(not np.array_equal(x, y) for i in range(4) for a, b in zip(tr.get_weights(i), plain.get_weights(i))
               for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------- agent API
@pytest.mark.parametrize("rule", ["clip", "scclip"])
def test_rpbcac_agent_methods_with_momentum(K, rule):
    """RPBCAC_agent(..., momentum=0.9): three rounds of hidden consensus, estimate consensus and projection step
    against the oracle agent fed the oracle's momentum rows (reference c = the agent's net at its hidden call; the
    estimates reuse the hidden call's rows), with the agent's state M against the oracle's.  The estimates before any
    hidden call, and a changed neighbour count, are refused."""
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H, beta = 1, 0.9
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule,
                      momentum=beta)
    with pytest.raises(K.L.RcmarlError, match="hidden consensus call"):
        ag.resilient_consensus_critic(s, [list(w[j][1]) for j in range(5)])
    ora = NG._oracle_agent(rule, w[0], 0.01, 0.9, H)
    rs = np.random.RandomState(8600)
    M = [None, None]
    for round_ in range(3):
        nbrs = [0, 1, 3, 2, 4]
        cmsgs = [[np.asarray(x) + rs.randn(*np.shape(x)).astype(f32) * 0.05 for x in w[j][1]] for j in nbrs]
        tmsgs = [[np.asarray(x) + rs.randn(*np.shape(x)).astype(f32) * 0.05 for x in w[j][2]] for j in nbrs]
        per = []
        for net, (msgs, mine) in enumerate(((cmsgs, ora.critic), (tmsgs, ora.TR))):
            X = np.stack([MO.AT.pack(m, f64) for m in msgs])
            rows, M[net] = MO.step(X, MO.AT.pack(mine, f64), M[net], beta, round_ == 0)
            per.append([MO.AT.unpack(rows[k], msgs[0]) for k in range(rows.shape[0])])
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
        close(ag._momentum_M[0].cpu().numpy()[:, :M[0].shape[1]], M[0], rtol=1e-3, atol=1e-5)
    with pytest.raises(K.L.RcmarlError, match="one state per slot"):
        ag.resilient_consensus_critic_hidden(cmsgs[:4])
