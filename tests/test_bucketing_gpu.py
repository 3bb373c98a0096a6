"""GPU parity of randomized bucketing (rcmarl_bucket_mix, include/rcmarl.h) against the oracle (tests/bucket_oracle.py):
the kernel at n_in 1..16 and several s over the C2, C3 and 16-agent widths in launches of 32 jobs, bitwise determinism
across calls, job orders and launch splits, the counter words, poisoned rows and the refusals; whole update rounds
through Trainer (C2 with agent 4 Byzantine under the 6 rules that accept 3 rows, a 16-agent team mixing nnm and
bucketing per agent), a world-1 PeerComm, the drop-in train_RPBCAC path and the per-agent API.

The permutation, the buckets and M must match exactly.  The kernel's bucket means must equal the fp32 oracle's bit
for bit (the same additions in the same order, then one division) and lie within 4e-6 max|x| of the fp64 ones (as
test_nnm_gpu.py).  After whole update rounds weights rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as
test_trainer_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                    # noqa: E402
import bucket_oracle as BO                             # noqa: E402
import dissensus_mimic_oracle as DM                    # noqa: E402
import nnm_oracle as NO                                # noqa: E402
import team_util as TU                                 # noqa: E402
import test_nnm_gpu as NG                              # noqa: E402  (the C2 round helpers)
from golden_util import load, pretrained               # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
RULES6 = ("clip", "trim", "wmsr", "scclip", "gmed", "dnc")      # the rules that accept 3 rows at H = 1
PAR_COUNTS = NG.PAR_COUNTS                                      # 5- / 16-agent critic / TR nets
S_VALUES = (1, 2, 3, 5, 16)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _outputs(K, n_jobs, stride):
    return (torch.full((n_jobs, 16, stride), NAN, device=K.dev), torch.full((n_jobs, 256), NAN, device=K.dev))


def _cases(rs, n_rows=24):
    """(n_in, s, P, nodes, (seed, receiver, net, round, epoch)) over n_in 1..16 and every s of S_VALUES."""
    out = []
    for n_in in range(1, 17):
        for q, s in enumerate(S_VALUES):
            nodes = [int(x) for x in rs.choice(n_rows, size=n_in, replace=False)]
            if n_in >= 3 and (n_in + q) % 3 == 1:
                nodes[-1] = nodes[int(rs.randint(0, n_in - 1))]                  # a repeated in-node
            words = (int(rs.randint(0, 2 ** 62)) * 3, int(rs.randint(0, 256)), int(rs.randint(0, 2)),
                     int(rs.randint(0, 2 ** 32, dtype=np.uint64)), int(rs.randint(0, 50)))
            out.append((n_in, s, PAR_COUNTS[(n_in + q) % 4], nodes, words))
    return out


def _job(K, dst, msgs, P, nodes, s, words, weights_out=None):
    seed, receiver, net, round_, epoch = words
    return K.ops.bucket_job(dst, msgs, msgs.shape[1], P, nodes, s, seed=seed, receiver=receiver, net=net, round=round_,
                            epoch=epoch, weights_out=weights_out)


def test_bucket_mix_against_the_oracle(K):
    """n_in 1..16, s in 1, 2, 3, 5, 16, the trainer's parameter counts, repeated in-nodes, launches of 32 jobs: M and the
    buckets exactly, the rows bitwise against fp32 and within tolerance of fp64, nothing written past n_out rows."""
    rs = np.random.RandomState(7100)
    stack = NG._stack(rs)
    msgs = to_dev(K, stack)[0]
    S = stack.shape[1]
    cases = _cases(rs)
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        dst, wout = _outputs(K, len(part), S)
        K.ops.bucket_mix([_job(K, dst[j, 0], msgs, P, nodes, s, words, weights_out=wout[j])
                          for j, (_, s, P, nodes, words) in enumerate(part)])
        got, gw = dst.cpu().numpy(), wout.cpu().numpy()
        for j, (n_in, s, P, nodes, words) in enumerate(part):
            n_out = BO.n_out(n_in, s)
            tag = f"n_in={n_in} s={s} P={P} nodes={nodes} words={words}"
            assert np.isnan(got[j, n_out:]).all() and np.isnan(got[j, :n_out, P:]).all(), f"{tag}: wrote past the rows"
            assert np.isnan(gw[j, n_out * n_in:]).all(), f"{tag}: wrote past n_out * n_in weights"
            X = stack[nodes, :P]
            want32, M32 = BO.bucket_mix(X, s, *words)
            want64, M64 = BO.bucket_mix(X.astype(f64), s, *words)
            M = gw[j, :n_out * n_in].reshape(n_out, n_in)
            np.testing.assert_array_equal(M, M32, err_msg=tag)
            np.testing.assert_array_equal(M, M64.astype(np.float32), err_msg=tag)
            np.testing.assert_array_equal(got[j, :n_out, :P], want32, err_msg=tag)
            close(got[j, :n_out, :P], want64, rtol=0, atol=NG.out_atol(np.abs(X).max()), err_msg=tag)


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(7200)
    stack = NG._stack(rs)
    msgs = to_dev(K, stack)[0]
    every = _cases(rs)
    cases = every[::5] + every[2::5]                                             # n_in 1 .. 16 twice, every s
    dst, wout = _outputs(K, len(cases), stack.shape[1])
    jobs = [_job(K, dst[j, 0], msgs, P, nodes, s, words, weights_out=wout[j])
            for j, (_, s, P, nodes, words) in enumerate(cases)]
    assert len(jobs) == 32 and {c[0] for c in cases} >= {1, 4, 16}

    def run(groups):
        dst.fill_(NAN)
        wout.fill_(NAN)
        for g in groups:
            K.ops.bucket_mix(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(wout, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_the_draws_change_with_every_counter_word(K):
    """One job at n_in = 16, s = 1 (M is the permutation) under each counter word and the seed moved by one."""
    rs = np.random.RandomState(7300)
    stack = NG._stack(rs, n_rows=16, P=700)
    msgs = to_dev(K, stack)[0]
    base = (11, 3, 0, 40, 2)
    variants = [base] + [tuple(v + 1 if q == k else v for q, v in enumerate(base)) for k in range(5)]
    dst, wout = _outputs(K, len(variants), 700)
    K.ops.bucket_mix([_job(K, dst[j, 0], msgs, 700, list(range(16)), 1, w, weights_out=wout[j])
                      for j, w in enumerate(variants)])
    gw = wout.cpu().numpy()[:, :256].reshape(-1, 16, 16)
    perms = {tuple(np.argmax(M[1:], 1)) for M in gw}
    assert len(perms) == len(variants)
    for j, w in enumerate(variants):
        assert list(np.argmax(gw[j][1:], 1)) == BO.permutation(16, *w)


@pytest.mark.parametrize("poison", [np.inf, -np.inf, 3e38, "pm"])
def test_poisoned_rows(K, poison):
    """H rows of +-inf, or of 3e38 (whose bucket sums overflow), give at most H bucket rows of +inf; +inf and -inf in
    one bucket give +inf, not NaN; every other row is the fp32 oracle's bit for bit."""
    rs = np.random.RandomState(7400)
    P = 761
    stack = NG._stack(rs, n_rows=24, P=P)
    bad_rows = list(range(16, 24))
    for q, r in enumerate(bad_rows):
        if poison == "pm":
            stack[r] = np.inf if q % 2 == 0 else -np.inf
        else:
            stack[r, ::3] = poison
    msgs = to_dev(K, stack)[0]
    cases = []
    for n_in, s, H in ((4, 2, 1), (8, 2, 2), (16, 3, 3), (9, 4, 2), (16, 1, 5), (16, 16, 4), (5, 2, 2)):
        bad = [int(x) for x in rs.choice(bad_rows, size=H, replace=False)]
        honest = [int(x) for x in rs.choice(16, size=n_in - 1 - H, replace=False)]
        cases.append((n_in, s, [int(rs.randint(16))] + [int(x) for x in rs.permutation(honest + bad)], H,
                      (int(rs.randint(1000)), n_in, 1, 5, 6)))
    dst, wout = _outputs(K, len(cases), P)
    K.ops.bucket_mix([_job(K, dst[j, 0], msgs, P, nodes, s, words, weights_out=wout[j])
                      for j, (_, s, nodes, _, words) in enumerate(cases)])
    got = dst.cpu().numpy()
    for j, (n_in, s, nodes, H, words) in enumerate(cases):
        n_out = BO.n_out(n_in, s)
        want, _ = BO.bucket_mix(stack[nodes], s, *words)
        np.testing.assert_array_equal(got[j, :n_out], want, err_msg=str(cases[j]))
        poisoned = [k for k in range(1, n_out) if not np.isfinite(got[j, k]).all()]
        assert len(poisoned) <= H and all((got[j, k] == np.inf).all() for k in poisoned), cases[j]
        if poison != 3e38:
            assert poisoned, cases[j]


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(7500)
    P = 700
    stack = NG._stack(rs, n_rows=8, P=P)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((3, 4, P), NAN, device=K.dev)
    wout = torch.full((3, 256), NAN, device=K.dev)
    B = K.ops.bucket_job
    good = B(dst[0, 0], msgs, P, P, [0, 1, 2, 3], 2, seed=1, weights_out=wout[0])
    d, w = dst[1, 0], wout[1]
    bad = [B(d, msgs, P, P, [0, 1, 2], 0, weights_out=w),                      # s < 1
           B(d, msgs, P, P, [0, 1, 2], -4, weights_out=w),
           B(d, msgs, P, P, [], 2, weights_out=w),
           B(d, msgs, P, P, list(range(8)) * 2 + [0], 2, weights_out=w),        # 17 in-nodes
           B(d, msgs, P, P, [0, -1, 2], 2, weights_out=w),
           B(d, msgs, P, P, [0, 1, 2], 2, net=2, weights_out=w),
           B(d, msgs, P, P, [0, 1, 2], 2, receiver=256, weights_out=w),
           B(d, msgs, P, 0, [0, 1, 2], 2, weights_out=w),
           B(msgs[2], msgs, P, P, [0, 1, 2], 2, weights_out=w),                 # dst row 0 is an in-node row
           B(msgs[5], msgs, P, P, [0, 1, 6], 1, weights_out=w),                 # dst row 1 is in-node row 6
           B(dst[0, 2], msgs, P, P, [5, 6, 7], 2, weights_out=w),               # dst rows on the other job's
           B(d, msgs, P, P, [0, 1, 2], 2, weights_out=msgs[1][5:]),             # weights_out on an in-node row
           B(d, msgs, P, P, [0, 1, 2], 2, weights_out=dst[0, 2][10:]),          # ... on the other job's dst row 2
           B(d, msgs, P, P, [0, 1, 2], 1, weights_out=dst[1, 2][3:]),           # ... on its own dst row 2
           B(d, msgs, P, P, [0, 1, 2], 2, weights_out=wout[0][11:]),            # ... on the other's weights_out
           B(d, msgs, P // 2, P // 2 + 1, [0, 1, 2], 1, weights_out=w)]         # its own dst rows overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.bucket_mix([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(wout).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.bucket_mix([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(wout).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an in-node row was written"
    K.ops.bucket_mix([good])
    assert torch.isfinite(dst[0, :3]).all() and torch.isfinite(wout[0, :12]).all() and torch.isnan(dst[0, 3]).all()
    assert torch.isnan(dst[1:]).all()


# ---------------------------------------------------------------------------------------------------------- Trainer
def _oracle_round(agents, labels, in_nodes, rows, inner, mixing, H, N, T, round_, seed, kernel_M=None, n_epochs=2):
    """The oracle's round with `inner` (an attack hook) inside nnm_oracle's hook for the nnm agents, inside the bucket
    hook for the bucketing agents."""
    log = {}
    nnm = [m if m == "nnm" else None for m in mixing]
    if any(nnm):
        inner = NO.mixing_hook(labels, in_nodes, nnm, H, inner=inner, kernel_M=kernel_M)
    hook = BO.bucketing_hook(labels, in_nodes, mixing, seed, round_, inner=inner, log=log)
    loss = NO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    return loss, log


def _check_bucket_M(tr, agents, rules, log):
    """Trainer.mixing_matrices of the bucketing agents against the oracle's last-epoch M exactly, and for the
    whole-message rules neighbour_weights against the oracle rule's weights times M."""
    mats = tr.mixing_matrices()
    got = tr.neighbour_weights()
    for i in log:
        n_in = len(tr.in_nodes[i])
        assert mats[i].shape == (2, BO.n_out(n_in, tr.mixing[i][1]), n_in)
        for t in range(2):
            np.testing.assert_array_equal(mats[i][t], log[i][-1][t][0].astype(np.float32), err_msg=f"agent {i} {t}")
        if rules[i] in ("krum", "mkrum", "scclip", "gmed"):
            rule_w = np.stack(agents[i].last_weights[-4:-2])
            for t in range(2):
                want = rule_w[t] @ log[i][-1][t][0]
                atol = 1e-7 if rules[i] in ("krum", "mkrum") else 2e-3
                close(got[i][t], want, rtol=1e-6, atol=atol, err_msg=f"agent {i} net {t}")
        if i in got:
            assert got[i].shape == (2, n_in)
            np.testing.assert_allclose(got[i].sum(1), 1.0, atol=1e-5)


ATTACKS = {"mimic": 1, "alie": 1.5}


@pytest.mark.parametrize("kind", list(ATTACKS))
@pytest.mark.parametrize("rule", RULES6)
def test_c2_update_round_with_a_byzantine_agent(K, rule, kind):
    """The benchmark's 5-agent team with agent 4 Byzantine, every cooperative agent bucketing (s = 2: its own row and
    2 bucket means) before `rule` (H = 1): two epochs against the oracle's round with the attack hook inside the bucket
    hook; one bucketing launch per epoch more than without bucketing."""
    w, desired, _ = pretrained()
    gamma, T, round_, N = 0.9, 40, 150, 64
    rs = np.random.RandomState(7600)
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule)
    mixing = [("bucket", 2)] * 4 + [None]
    tr, got, _, runs = NG._kernel_M(cfg, rows, round_, "bucket")
    assert tr.mixing == mixing
    agents = [NG._oracle_agent(rule, w[i], 0.01, gamma, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    NG._follow_dnc(agents, runs)
    inner = DM.StateHook(C2_BYZ, IN_NODES, {4: attack}, [rule] * 5, [1] * 5, seed=9, round_=round_, gap=1e-4)
    inner.follow = {e: r.mimic_targets() for e, r in enumerate(runs)}
    want, log = _oracle_round(agents, C2_BYZ, IN_NODES, rows, inner, mixing, [1] * 5, N, T, round_, seed=9)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    assert sorted(log) == tr.mix_agents == [0, 1, 2, 3]
    _check_bucket_M(tr, agents, [rule] * 5, log)
    plain, _ = NG._trainer_round(cfg, rows, round_, 2, None)
    assert tr.launches - plain.launches == 2                                    # one bucketing launch per epoch
    assert tr.msg_c.shape[0] - plain.msg_c.shape[0] == 4 * 3                    # n_out = 3 rows per agent


RULES16 = ["dnc", "clip", "gmed", "trim", "mkrum", "wmsr", "scclip", "krum"]   # the 8 cooperative agents, in order
MIX16 = [("bucket", 2), "nnm", None, ("bucket", 2), ("bucket", 2), "nnm", ("bucket", 3), ("bucket", 2)]


def test_16_agent_team_with_nnm_and_bucketing(K):
    """16 agents (8 cooperative, 5 Byzantine with mixed attacks, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, receiver
    0 listing Byzantine agent 1 twice) with the cooperative agents' rules and mixing set per agent: Krum and multi-Krum
    bucket (5 rows at s = 2), and receiver 0's doubled Byzantine entry lands in its buckets twice."""
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
            agents.append(NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[attacks.get(i) for i in range(16)])
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    NG._follow_dnc(agents, runs)
    inner = AA.make_hook(labels, in_nodes, attacks, seed=4, round_=round_)
    want, log = _oracle_round(agents, labels, in_nodes, rows, inner, mixing, H, N, T, round_, seed=4,
                              kernel_M=kernel_M)
    n_bucket = sum(m is not None and m != "nnm" for m in MIX16)
    assert tr.mix_agents == [i for i in coop if mixing[i] is not None]
    assert tr.msg_c.shape[0] == 16 + len(tr.byz_pairs) + 4 + 1 + 2 * 8 + (n_bucket - 1) * 5 + 4
    assert in_nodes[0].count(1) == 2 and mixing[0] == ("bucket", 2)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]}, {mixing[i]})")
    _check_bucket_M(tr, agents, rules, log)


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


def test_world1_peer_comm_with_bucketing_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run whose agents bucket."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["dnc", "scclip", "trim", "clip", "clip"],
                     mixing=["bucket", ("bucket", 1), "nnm", None, None], attack=("mimic", 3))
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append(NG._state(tr))
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_train_rpbcac_with_bucketing_and_nnm_agents(K):
    """Drop-in path: train_RPBCAC with RPBCAC_agent objects that bucket or mix runs the same round as a Trainer built
    from the same objects with the same mixing passed directly, bit for bit, and differs from a run without mixing."""
    import contextlib
    import io
    from rcmarl import api
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)
    mixing = [("bucket", 2), "nnm", None, "bucket", None]

    def objects(with_mixing):
        env, agents, args = api.build_reference_objects(cfg)
        if with_mixing:
            for i in range(4):
                agents[i].mixing = K.L.mixing_entry(mixing[i])
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    env, agents, args = objects(True)
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(env, agents, args)
    tr = training.train_RPBCAC.last_trainer
    assert tr.mixing == [("bucket", 2), "nnm", None, ("bucket", 2), None] and tr.mix_agents == [0, 1, 3]
    env2, agents2, args2 = objects(False)
    direct = training.build_trainer(env2, agents2, args2, mixing=mixing)
    plain = training.build_trainer(*objects(False))
    for t in (direct, plain):
        for _ in range(2):
            t.rollout_block(4)
            t.update_round()
    torch.cuda.synchronize()
    assert direct.launches == tr.launches == plain.launches + 2 * 2 * 2      # nnm + bucketing launch per epoch
    for i in range(5):
        for a, b in zip(tr.get_weights(i), direct.get_weights(i)):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
    assert any(not np.array_equal(x, y) for i in range(4) for a, b in zip(tr.get_weights(i), plain.get_weights(i))
               for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------- agent API
@pytest.mark.parametrize("rule", ["clip", "scclip"])
def test_rpbcac_agent_methods_with_bucketing(K, rule):
    """RPBCAC_agent(..., mixing=("bucket", 2)) keyed by the facade seed: two rounds of hidden consensus, estimate
    consensus and projection step (round = the per-net hidden call count; the estimates reuse the last hidden call's
    buckets), and _resilient_aggregation (net 0, round 0), against the oracle agent fed the oracle's bucket rows."""
    import tensorflow as tf
    from agents.resilient_CAC_agents import RPBCAC_agent
    from test_aggregation_rules_gpu import build_models
    z = load("ref_methods.npz")
    w, _, _ = pretrained()
    s, a = z["s"], z["a"]
    sa = np.concatenate([s, a], -1)
    H, seed = 1, 123457
    tf.random.set_seed(seed)
    ag = RPBCAC_agent(*build_models(w[0]), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=H, aggregation=rule,
                      mixing=("bucket", 2))
    tf.random.set_seed(0)                                   # the agent keeps the seed it was built under
    ora = NG._oracle_agent(rule, w[0], 0.01, 0.9, H)
    nbrs = [0, 1, 3, 2, 4]
    cmsgs = [list(w[j][1]) for j in nbrs]
    tmsgs = [list(w[j][2]) for j in nbrs]
    for round_ in range(2):
        hook = BO.bucketing_hook(["Cooperative"], [[0]], [("bucket", 2)], seed, round_,
                                 inner=lambda e, c, t: ({0: c}, {0: t}))
        mc, mt = hook(0, cmsgs, tmsgs)
        mc, mt = mc[0], mt[0]
        assert len(mc) == len(mt) == 3
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
    Y, _ = BO.bucket_mix(v.reshape(7, -1).astype(f64), 2, seed, 0, 0, 0, 0)
    want = NG.AO.resilient_aggregation(Y, H, "clip") if rule == "clip" else NG.VO.aggregate(Y, H, rule)[0]
    close(ag._resilient_aggregation(v).numpy(), want.reshape(3, 11), rtol=0, atol=NG.out_atol(np.abs(v).max()))
    with pytest.raises(K.L.RcmarlError):
        ag.H = 7                                            # H < n_in = 7
        ag._resilient_aggregation(v)
