"""GPU parity of the Byzantine attacks (rcmarl_attack, include/rcmarl.h) against the float64 oracle
(tests/attack_oracle.py): the kernel with the three kinds mixed in one launch, whole update rounds through Trainer with
per-receiver crafted messages under each aggregation rule, a 16-agent team whose attack jobs run in groups, checkpoint
resume, the data-parallel paths that run on one GPU, the refusals, and the unchanged default.

Tolerances: the kernel as rcmarl_clip_mean's test (atol 4e-6 max|v|), scaled by (1 + |param|); weights after whole
update rounds rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as test_trainer_gpu.py)."""
import datetime
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import agg_oracle as AO                                # noqa: E402
import attack_oracle as AT                             # noqa: E402
import team_util as TU                                 # noqa: E402
from golden_util import pretrained                     # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
C2_BYZ = ["Cooperative"] * 4 + ["Byzantine"]
PARAMS = {"alie": 1.5, "ipm": 0.5, "gauss": 0.3}
PAR_COUNTS = (661, 761, 1101, 1421, 300)              # 5- / 16-agent critic / TR nets, and a short ragged one


@pytest.fixture(scope="module")
def K():
    return load_kernels()


# ---------------------------------------------------------------------------------------------------------- kernel
def _kernel_case(K, seed=2100):
    """32 jobs: kinds cycling, n_honest 1..16 with repeated indices, the parameter counts above; per job the fp64
    oracle's message."""
    rs = np.random.RandomState(seed)
    n_rows, P = 20, max(PAR_COUNTS)
    stack = (rs.randn(n_rows, P) * rs.uniform(0.1, 3, size=(n_rows, 1))).astype(np.float32)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((32, P), float("nan"), device=K.dev)
    jobs, want, spec = [], [], []
    for j in range(32):
        kind = AT.ATTACKS[j % 3]
        n_h = j % 16 + 1
        honest = [int(x) for x in rs.randint(0, n_rows, size=n_h)]
        if n_h >= 3:
            honest[-1] = honest[0]                                           # a repeated index
        n = PAR_COUNTS[j % len(PAR_COUNTS)]
        param = float([1.5, -0.7, 3.0, 0.0, 0.25][j % 5]) if kind != "gauss" else float([0.3, 0.0, 2.0][j // 3 % 3])
        ctr = dict(seed=(7 << 32) + 123 + j % 2, attacker=j % 7, receiver=(j * 5) % 16, round=1000 + j % 3, epoch=j % 4)
        jobs.append(K.ops.attack_job(dst[j], msgs, P, n, honest, kind, param, **ctr))
        vals = stack[honest, :n].astype(np.float64)
        xi = AT.gauss_xi(n, ctr["seed"], ctr["attacker"], ctr["receiver"], ctr["round"], ctr["epoch"]) if kind == "gauss" else None
        want.append(AT.craft(vals, kind, param, xi))
        spec.append((kind, param, n, np.abs(vals).max()))
    return msgs, dst, jobs, want, spec


def test_attack_kinds_mixed_in_one_launch(K):
    msgs, dst, jobs, want, spec = _kernel_case(K)
    K.ops.attack(jobs)
    got = dst.cpu().numpy()
    for j, ((kind, param, n, vmax), w) in enumerate(zip(spec, want)):
        close(got[j, :n], w, rtol=0, atol=4e-6 * max(vmax, 1.0) * (1 + abs(param)), err_msg=f"job {j} {kind} {param}")
        assert np.isnan(got[j, n:]).all(), f"job {j} wrote past n"


def test_attack_is_bitwise_deterministic_across_calls_orders_and_splits(K):
    msgs, dst, jobs, _, _ = _kernel_case(K)
    K.ops.attack(jobs)
    first = dst.clone()
    dst.fill_(float("nan"))
    K.ops.attack(jobs)
    assert torch.equal(torch.nan_to_num(dst, 7.0), torch.nan_to_num(first, 7.0))
    dst.fill_(float("nan"))
    K.ops.attack(jobs[::-1])
    assert torch.equal(torch.nan_to_num(dst, 7.0), torch.nan_to_num(first, 7.0))
    dst.fill_(float("nan"))
    for g in (jobs[5:9], jobs[:5], jobs[9:]):
        K.ops.attack(g)
    assert torch.equal(torch.nan_to_num(dst, 7.0), torch.nan_to_num(first, 7.0))


def test_attack_refusals_leave_dst_untouched(K):
    msgs, dst, jobs, _, _ = _kernel_case(K)
    before = dst.clone()
    P = msgs.shape[1]
    d, m = dst[1], msgs
    bad = [K.ops.attack_job(d, m, P, 0, [0, 1], "alie", 1.0),
           K.ops.attack_job(d, m, P, 10, [], "alie", 1.0),
           K.ops.attack_job(d, m, P, 10, list(range(17)), "ipm", 1.0),
           K.ops.attack_job(d, m, P, 10, [0, -2], "ipm", 1.0),
           K.ops.attack_job(d, m, P, 10, [0, 1], 5, 1.0),
           K.ops.attack_job(d, m, P, 10, [0, 1], "alie", float("nan")),
           K.ops.attack_job(d, m, P, 10, [0, 1], "ipm", float("inf")),
           K.ops.attack_job(d, m, P, 10, [0, 1], "gauss", -1.0),
           K.ops.attack_job(d, m, P, 10, [0, 1], "gauss", 1.0, receiver=256)]
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.attack([jobs[0], b])
        torch.cuda.synchronize()
        assert torch.equal(torch.nan_to_num(dst, 7.0), torch.nan_to_num(before, 7.0))
    with pytest.raises(K.L.RcmarlError):
        K.ops.attack_job(d, m, P, 10, [0, 1], "median", 1.0)
    with pytest.raises(K.L.RcmarlError):
        K.ops.attack(jobs + jobs[:1])                                        # 33 jobs


# ---------------------------------------------------------------------------------------------------------- Trainer
def _c2_agents(w, rule, gamma):
    ags = [AO.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, 0.01, gamma, H=1, dtype=np.float64, aggregation=rule)
           for i in range(4)]
    ags.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=np.float64))
    return ags


def _oracle_round(agents, labels, in_nodes, rows, attacks, N, T, round_, seed=0, n_epochs=2, crafted=True):
    prs = np.random.RandomState(1700)
    used = []

    def rec(T_):
        p = prs.permutation(T_)
        used.append(p)
        return p
    hook = AT.make_hook(labels, in_nodes, attacks, seed=seed, round_=round_) if crafted else None
    loss = AT.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=rec, messages_hook=hook)
    return loss, used


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("rule", ["clip", "trim", "wmsr"])
@pytest.mark.parametrize("kind", AT.ATTACKS)
def test_c2_update_round_with_a_byzantine_agent(K, kind, rule, N):
    """The benchmark's 5-agent team with agent 4 Byzantine: one update round of two epochs (the messages are crafted
    anew in each) against the oracle's round with the per-receiver hook."""
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(2200 + N)
    rows = synth(rs, T * N)
    attack = (kind, PARAMS[kind])
    agents = _c2_agents(w, rule, gamma)
    want, used = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: attack}, N, T, round_, seed=9)
    it = iter(list(used))
    tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
                 slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=9, aggregation=rule,
                 attack=attack, perm_source=lambda T_: next(it))
    assert [(b, j) for b, j, _ in tr.byz_pairs] == [(4, 1), (4, 2), (4, 3)]
    tr.load_rows(*rows)
    tr.episodes_done = round_
    got = tr.update_round()
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")


B16 = ["Cooperative", "Byzantine", "Cooperative", "Malicious", "Cooperative", "Byzantine", "Cooperative", "Greedy",
       "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Malicious", "Byzantine", "Cooperative"]


def _team16(rs):
    """16 agents on the 10x10 grid: 8 cooperative, 5 Byzantine with mixed attacks, 2 Malicious, 1 Greedy; circulant
    in-neighbourhoods of 8 (19 attacker-receiver pairs, 38 attack jobs), and receiver 0 lists Byzantine agent 1 twice."""
    from rcmarl import nets
    NA = 16
    in_nodes = [[(i + k) % NA for k in range(8)] for i in range(NA)]
    in_nodes[0] = [0, 1, 2, 3, 1, 5, 6, 7]
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    for i in range(NA):
        if B16[i] == "Malicious":
            w[i].append(nets.glorot_uniform(32, 1, rs))
    attacks = {1: ("alie", 1.0), 5: ("gauss", 0.5), 9: ("ipm", 0.25), 11: ("alie", -0.5), 14: ("gauss", 0.0)}
    return in_nodes, w, rs.randint(0, 10, size=(NA, 2)), [i % 3 for i in range(NA)], [0.01 + 0.001 * (i % 4) for i in range(NA)], attacks


@pytest.mark.parametrize("rule", ["clip", "wmsr"])
def test_16_agent_team_with_several_byzantine_agents(K, rule):
    """More than 32 (attacker, receiver, net) jobs, so the attack launches run in groups; a receiver that lists the
    same attacker twice gets its one crafted message twice."""
    from rcmarl.trainer import Trainer
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, attacks = _team16(rs)
    gamma, T, N, round_ = 0.9, 40, 4, 7
    pairs = AT.byzantine_pairs(B16, in_nodes)
    assert 2 * len(pairs) > 32 and in_nodes[0].count(1) == 2
    agents = []
    for i, lab in enumerate(B16):
        if lab == "Cooperative":
            agents.append(AO.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, fast[i], gamma, H=H[i], dtype=np.float64,
                                               aggregation=rule))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    want, used = _oracle_round(agents, B16, in_nodes, rows, attacks, N, T, round_, seed=4)
    it = iter(list(used))
    tr = Trainer(labels=B16, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma, H=H,
                 fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=4,
                 aggregation=rule, attack=[attacks.get(i) for i in range(16)], perm_source=lambda T_: next(it))
    assert [(b, j) for b, j, _ in tr.byz_pairs] == [(b, j) for b, j, _ in pairs]
    tr.load_rows(*rows)
    tr.episodes_done = round_
    launches = tr.launches
    got = tr.update_round()
    n_groups = (2 * len(pairs) + 31) // 32
    assert n_groups >= 2
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({B16[i]})")
    # the same team with Faulty agents in place of the Byzantine ones makes n_groups fewer launches per epoch
    labels_f = ["Faulty" if l == "Byzantine" else l for l in B16]
    it = iter(list(used))
    tf = Trainer(labels=labels_f, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
                 H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=4,
                 aggregation=rule, perm_source=lambda T_: next(it))
    tf.load_rows(*rows)
    tf.update_round()
    assert (tr.launches - launches) - tf.launches == 2 * n_groups


def _c2_trainer(attack, labels=C2_BYZ, **kw):
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    cfg = dict(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=16, gamma=0.9, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21, attack=attack)
    cfg.update(kw)
    return Trainer(**cfg)


def _state(tr):
    return [getattr(tr, n).clone() for n in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v")]


def test_checkpoint_resume_with_gauss_is_bitwise(K, tmp_path):
    """save after round 1 and load into a fresh Trainer: round 2 (Philox rollout + update with a gauss attacker, whose
    draws are keyed by episodes_done) equals the uninterrupted run bit for bit."""
    ref = _c2_trainer(("gauss", 0.4))
    for _ in range(2):
        ref.rollout_block()
        ref.update_round()
    a = _c2_trainer(("gauss", 0.4))
    a.rollout_block()
    a.update_round()
    a.save(tmp_path / "ck.pt")
    b = _c2_trainer(("gauss", 0.4))
    b.load(tmp_path / "ck.pt")
    b.rollout_block()
    b.update_round()
    torch.cuda.synchronize()
    for x, y in zip(_state(b), _state(ref)):
        assert torch.equal(x, y)
    # and the round counter matters: the same run with round 2 keyed as round 1 differs
    c = _c2_trainer(("gauss", 0.4))
    c.load(tmp_path / "ck.pt")
    c.rollout_block()
    c.episodes_done -= c.n_ep_fixed
    c.update_round()
    assert not torch.equal(c.critic, ref.critic)


def test_trainer_refusal_leaves_weights_untouched(K):
    """A bad attack is refused when the Trainer is built; a Trainer whose attack job table is made invalid afterwards
    refuses in update_round before the attack launch writes anything."""
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        _c2_trainer(("gauss", -1.0))
    tr = _c2_trainer(("alie", 1.0))
    tr.rollout_block()
    before = _state(tr)
    msg_before = (tr.msg_c[5:].clone(), tr.msg_t[5:].clone())
    tr.attack[4] = (7, 1.0)                                                 # an unknown kind reaches the library
    with pytest.raises(L.RcmarlError):
        tr.update_round()
    torch.cuda.synchronize()
    assert torch.equal(tr.msg_c[5:], msg_before[0]) and torch.equal(tr.msg_t[5:], msg_before[1])
    assert all(torch.equal(x, y) for x, y in zip(_state(tr), before))       # Phase I writes only the message rows


def test_default_is_unchanged(K):
    """Without a Byzantine agent the Trainer issues the calls it always did: attack=None and one None per agent are
    bitwise equal, with the same launch count; a Byzantine agent only adds the attack launches to a Faulty one's."""
    runs = []
    for attack in (None, [None] * 5):
        tr = _c2_trainer(attack, labels=pretrained()[2])
        tr.rollout_block()
        tr.update_round()
        runs.append((tr.launches, _state(tr), tr.msg_c.shape[0]))
    assert runs[0][0] == runs[1][0] and runs[0][2] == runs[1][2] == 5
    assert all(torch.equal(x, y) for x, y in zip(runs[0][1], runs[1][1]))
    f = _c2_trainer(None, labels=["Cooperative"] * 4 + ["Faulty"])
    b = _c2_trainer(("ipm", 1.0))
    for t in (f, b):
        t.rollout_block()
        t.update_round()
    assert b.launches - f.launches == b.n_epochs and b.msg_c.shape[0] == 5 + 3
    assert torch.equal(b.actor[4], f.actor[4])                              # the attacker learns like a Faulty agent
    assert not torch.equal(b.critic[:4], f.critic[:4])


# ---------------------------------------------------------------------------------------------------------- data parallel
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


def test_world1_peer_comm_with_a_gauss_attacker_is_bitwise(K, gloo_world1):
    from rcmarl.comm import PeerComm
    runs = []
    for bound in (False, True):
        tr = _c2_trainer(("gauss", 0.3), n_envs=64)
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append(_state(tr))
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_two_ranks_with_a_gauss_attacker_match_the_oracle(K, tmp_path):
    """2 ranks x 4 environments over gloo with RCMARL_PEER_COMM=0 (test_dp_single_gpu.py's worker): the ranks'
    parameters are bitwise equal and match the oracle's round with the per-receiver hook over all 8 environments."""
    import torch.multiprocessing as mp
    import test_dp_single_gpu as DP
    w, desired, _ = pretrained()
    N, T = 8, 40
    team = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=[1] * 5,
                fast_lr=[0.01] * 5, attack=("gauss", 0.3))
    rs = np.random.RandomState(8)
    agents = TU.oracle_agents(C2_BYZ, w, team["H"], team["fast_lr"], DP.COMMON["gamma"])
    rows, perms, losses = [], [], []
    for _ in range(2):
        data = TU.grid_rows(rs, T * N, 5, 5)
        buf = data if not rows else tuple(np.concatenate([x, y])[-DP.COMMON["buffer_size"] * N:] for x, y in zip(rows[-1][1], data))
        loss, used = _oracle_round(agents, C2_BYZ, IN_NODES, buf, {4: team["attack"]}, N,
                                   DP.COMMON["max_ep_len"] * DP.COMMON["n_ep_fixed"], 0, n_epochs=DP.COMMON["n_epochs"])
        rows.append((data, buf))
        perms.append(used)
        losses.append(loss)
    case = dict(kind="injected", team=team, N=N, rows=[r[0] for r in rows], perms=perms)
    mp.spawn(DP._worker, args=(2, str(tmp_path / "pg"), {"byz": case}, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = DP._load_ranks(tmp_path, "byz")
    assert np.array_equal(r0["packed"], r1["packed"]), "replicated parameters diverged between ranks"
    for k, want in enumerate(losses):
        for key in ("critic_loss", "TR_loss", "actor_loss"):
            np.testing.assert_allclose(r0[f"r{k}_{key}"], want[key], rtol=2e-3, atol=2e-5, err_msg=f"round {k} {key}")
    got = DP._weights_of(r0, [len(ag.get_parameters()) for ag in agents])
    for i, ag in enumerate(agents):
        TU.close_w(got[i], ag.get_parameters(), msg=f"agent {i}")
