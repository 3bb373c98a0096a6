"""GPU parity of the pipeline-aware Byzantine messages (rcmarl_pipeline_attack, include/rcmarl.h) against the oracle
(tests/pipeline_attack_oracle.py): bitwise equality with rcmarl_tailored_attack without mixing for every coordinate-wise
and distance-based rule x direction at n_in 2..16; every family x mixing x direction against the fp64 oracle; model_out
against the real chain (rcmarl_nnm_mix, then rcmarl_vector_aggregate / rcmarl_dnc_aggregate / rcmarl_consensus_hidden)
run on the message stack with the crafted message written in; bitwise determinism across calls, job orders and launch
splits; the staging bound; whole update rounds through Trainer (C2 with agent 4 on pipeline_std under dnc, nnm + clip
and bucket + trim, a 16-agent team with colluding pipeline attackers and mixed rules, a world-1 PeerComm) and the
drop-in train_RPBCAC path.

Margins are handled as in test_tailored_attacks_gpu.py: where the oracle's relative margin between its best and its
second-best distinct mean objective exceeds MARGIN = 1e-4 the kernel's pick must be the oracle's, and otherwise the
fp64 objective of the kernel's pick must lie within MARGIN relative of the maximum.  In whole rounds the oracle's
attacker follows the kernel's pick at such a near tie (and the oracle's nnm receivers the kernel's selections, as in
test_nnm_gpu.py), since a near tie broken the other way moves the message by a whole candidate step."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                     # noqa: E402
import bucket_oracle as BO                              # noqa: E402
import nnm_oracle as NO                                 # noqa: E402
import pipeline_attack_oracle as PA                     # noqa: E402
import tailored_attack_oracle as TA                     # noqa: E402
import team_util as TU                                  # noqa: E402
import test_nnm_gpu as NG                               # noqa: E402  (the C2 round helpers)
import test_tailored_attacks_gpu as TG                  # noqa: E402  (the message stacks and cases)
from golden_util import pretrained                      # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                   # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = TG.IN_NODES
C2_BYZ = TG.C2_BYZ
PAR_COUNTS = TG.PAR_COUNTS
MARGIN = TG.MARGIN
MIXINGS = (None, "nnm", ("bucket", 2), ("bucket", 3))
WORDS = dict(seed=2 ** 40 + 77, attacker=9, receiver=3, net=1, round_=123, epoch=4)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _job(K, dst, msgs, case, scale, gamma_out=None, model_out=None, n_perms=3, words=WORDS):
    attack, rule, H, slots, honest, P, mixing = case
    w = dict(words)
    w["round"] = w.pop("round_")
    return K.ops.pipeline_attack_job(dst, msgs, msgs.shape[1], P, slots, honest, rule, H, attack, scale, mixing=mixing,
                                     n_perms=n_perms, gamma_out=gamma_out, model_out=model_out, **w)


def _max_h(rule, n):
    return 0 if n < 2 else TG._max_h(rule, n) if rule != "dnc" else n - 1


def _cases(rs, n_rows):
    """(attack, rule, H, slots, honest, P, mixing) for every rule (DnC included) x direction x mixing, n_in 2..16."""
    out = []
    base = TG._cases(rs, n_rows)                       # every coordinate-wise / distance-based rule x direction x n_in
    extra = [(a, "dnc", H, s, h, P) for (a, r, H, s, h, P) in base if r == "gmed"]
    for c, (attack, rule, H, slots, honest, P) in enumerate(base + extra):
        mixing = MIXINGS[c % 4]
        n_rows_rule = PA.n_rows(len(slots), mixing)
        if rule in ("krum", "mkrum") and n_rows_rule < 3:
            mixing = None if len(slots) >= 3 else mixing
            n_rows_rule = PA.n_rows(len(slots), mixing)
            if n_rows_rule < 3:
                continue
        H = min(H, _max_h(rule, n_rows_rule))
        out.append(("pipeline_" + attack.split("_")[1], rule, H, slots, honest, P, mixing))
    return out


def _check(got, gg, stack, case, scale, stats, words=WORDS, n_perms=3):
    attack, rule, H, slots, honest, P, mixing = case
    rows = stack[:, :P].astype(f64)
    want, g, Ob, _ = PA.craft(rows, slots, honest, rule, H, attack, scale, mixing=mixing, n_perms=n_perms, **words)
    V = np.stack([rows[slots[k]] for k in honest])
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    G = scale * g_mm
    tag = f"{attack} {rule} H={H} mixing={mixing} slots={slots} P={P}"
    assert np.isnan(got[P:]).all(), f"{tag}: wrote past n"
    i_gpu = 0 if G == 0 else int(round(float(gg) / G * PA.STEPS))
    if G != 0:
        close(gg, G * i_gpu / PA.STEPS, rtol=TG.G_RTOL, atol=0, err_msg=tag)
    m = PA.margin(Ob)
    if m > MARGIN:
        assert i_gpu == int(np.argmax(Ob)), f"{tag}: picked {i_gpu}, oracle {int(np.argmax(Ob))} (margin {m:.3g})"
        stats["exact"] += 1
    else:
        top = Ob.max()
        assert Ob[i_gpu] >= top - MARGIN * abs(top), f"{tag}: Obar[{i_gpu}] = {Ob[i_gpu]} vs max {top}"
        stats["near"] += 1
    gi = G * i_gpu / PA.STEPS
    close(got[:P], TA.candidate(mu, d, gi), rtol=0, atol=TG.msg_atol(np.abs(V).max(), gi, np.abs(d).max()), err_msg=tag)
    stats["interior"] += 0 < i_gpu < PA.STEPS


def test_without_mixing_bitwise_the_tailored_attack(K):
    """Every coordinate-wise and distance-based rule x direction at n_in 2..16: dst and gamma_out bit for bit."""
    rs = np.random.RandomState(8100)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = TG._cases(rs, stack.shape[0])
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        dst, gam, jobs = TG._launch(K, msgs, stack.shape[1], part, 2.0)
        K.ops.tailored_attack(jobs)
        pdst, pgam = torch.full_like(dst, NAN), torch.full_like(gam, NAN)
        K.ops.pipeline_attack([_job(K, pdst[j], msgs, (a.replace("tailored", "pipeline"), r, H, s, h, P, None), 2.0,
                                    gamma_out=pgam[j, :1]) for j, (a, r, H, s, h, P) in enumerate(part)])
        torch.cuda.synchronize()
        assert torch.equal(torch.nan_to_num(dst, 7.0), torch.nan_to_num(pdst, 7.0))
        assert torch.equal(torch.nan_to_num(gam, 7.0), torch.nan_to_num(pgam, 7.0))


def test_pipeline_attack_against_the_oracle(K):
    """Every family x mixing x direction at n_in 2..16 with 1-3 crafted and some Malicious-style real slots: the pick,
    gamma_out and the message against the fp64 oracle."""
    rs = np.random.RandomState(8200)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])
    assert {c[1] for c in cases} == set(PA.RULES) and {str(c[6]) for c in cases} == {str(m) for m in MIXINGS}
    stats = dict(exact=0, near=0, interior=0)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
        gam = torch.full((len(part), 2), NAN, device=K.dev)
        K.ops.pipeline_attack([_job(K, dst[j], msgs, c, 2.0, gamma_out=gam[j, :1]) for j, c in enumerate(part)])
        got, gg = dst.cpu().numpy(), gam.cpu().numpy()
        assert np.isnan(gg[:, 1]).all()
        for j, case in enumerate(part):
            _check(got[j], gg[j, 0], stack, case, 2.0, stats)
    print(f"{len(cases)} jobs: {stats}")
    assert stats["exact"] > len(cases) // 2 and stats["interior"] > 0


def _chain(K, msgs, stride, case, dst, model, coord_n):
    """The receiver's real chain on the stack with the crafted message dst written into every crafted slot: its mixed
    rows (rcmarl_nnm_mix) and its rule's output, compared with model_out bit for bit."""
    attack, rule, H, slots, honest, P, mixing = case
    n_rows = msgs.shape[0]
    stack = torch.cat([msgs, dst[None]])
    nodes = [n_rows if s < 0 else s for s in slots]
    if mixing == "nnm":
        mixed = torch.full((len(slots), stride), NAN, device=K.dev)
        K.ops.nnm_mix([K.ops.vector_job(mixed, stack, stride, P, nodes, H, K.L.MIX_NNM)])
        stack, nodes = mixed, list(range(len(slots)))
    out = torch.full((stride,), NAN, device=K.dev)
    if rule == "dnc":
        K.ops.dnc_aggregate([K.ops.vector_job(out, stack, stride, P, nodes, H, K.L.SPECTRAL_DNC)])
    elif rule in ("krum", "mkrum", "scclip", "gmed"):
        K.ops.vector_aggregate([K.ops.vector_job(out, stack, stride, P, nodes, H, rule)])
    else:
        K.ops.consensus_hidden([K.ops.consensus_job(out, stack, stride, P, nodes, H, rule)])
    torch.cuda.synchronize()
    a, b = out[:P].cpu().numpy(), model[:P].cpu().numpy()
    assert a.view(np.uint32).tolist() == b.view(np.uint32).tolist(), case


def test_model_out_is_the_real_chain_bitwise(K):
    """model_out against rcmarl_nnm_mix then the receiver's rule (rcmarl_vector_aggregate, rcmarl_dnc_aggregate, or
    rcmarl_consensus_hidden over every parameter for the coordinate-wise rules) on the message stack with the crafted
    message written in."""
    rs = np.random.RandomState(8300)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = [c for c in _cases(rs, stack.shape[0]) if c[6] in (None, "nnm")][::3][:32]
    assert {c[1] for c in cases} == set(PA.RULES) and {c[6] for c in cases} == {None, "nnm"}
    stride = stack.shape[1]
    dst = torch.full((len(cases), stride), NAN, device=K.dev)
    model = torch.full((len(cases), stride), NAN, device=K.dev)
    K.ops.pipeline_attack([_job(K, dst[j], msgs, c, 2.0, model_out=model[j]) for j, c in enumerate(cases)])
    torch.cuda.synchronize()
    for j, case in enumerate(cases):
        assert torch.isnan(model[j, case[5]:]).all()
        _chain(K, msgs, stride, case, dst[j], model[j], case[5])


def test_model_out_under_bucketing_is_sample_zero(K):
    """Under bucketing model_out is the rule on sample 0's rows: the fp32 oracle's rows and rule give it within fp32
    rounding."""
    rs = np.random.RandomState(8350)
    stack = TG._stack(rs, n_bad=0)
    msgs = to_dev(K, stack)[0]
    cases = [c for c in _cases(rs, stack.shape[0]) if isinstance(c[6], tuple) and c[1] in ("clip", "trim", "wmsr")][:16]
    stride = stack.shape[1]
    dst = torch.full((len(cases), stride), NAN, device=K.dev)
    model = torch.full((len(cases), stride), NAN, device=K.dev)
    K.ops.pipeline_attack([_job(K, dst[j], msgs, c, 1.0, model_out=model[j]) for j, c in enumerate(cases)])
    d, mo = dst.cpu().numpy(), model.cpu().numpy()
    for j, (attack, rule, H, slots, honest, P, mixing) in enumerate(cases):
        X = np.stack([d[j, :P] if s < 0 else stack[s, :P] for s in slots])
        bks = PA.buckets(len(slots), mixing[1], WORDS["seed"], 0, *[WORDS[k] for k in
                                                                    ("attacker", "receiver", "net", "round_", "epoch")])
        want = PA.rule_output(BO.mix(X, bks)[0], rule, H)
        close(mo[j, :P], want, rtol=1e-5, atol=1e-6, err_msg=f"{rule} {mixing} {slots}")


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(8400)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])[1::4][:32]
    assert len(cases) == 32
    dst = torch.full((32, stack.shape[1]), NAN, device=K.dev)
    gam = torch.full((32, 1), NAN, device=K.dev)
    model = torch.full((32, stack.shape[1]), NAN, device=K.dev)
    jobs = [_job(K, dst[j], msgs, c, 2.0, gamma_out=gam[j], model_out=model[j]) for j, c in enumerate(cases)]

    def run(groups):
        for t in (dst, gam, model):
            t.fill_(NAN)
        for g in groups:
            K.ops.pipeline_attack(g)
        return [torch.nan_to_num(t, 7.0).clone() for t in (dst, gam, model)]
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert all(torch.equal(a, b) for a, b in zip(again, first))


def test_staging_bound_and_refusals(K):
    """The 16-agent team-reward net (1421 parameters) at n_in = 16 under nnm with DnC, one crafted slot: exactly
    RCMARL_PIPELINE_MAX_FLOATS, accepted and run against the oracle; one parameter more (a row of floats past the
    bound) refused with every output untouched."""
    rs = np.random.RandomState(8500)
    P = 1421
    assert (15 + 16 + 4 + 2) * P == K.L.PIPELINE_MAX_FLOATS
    X = (rs.randn(16, P + 1) * rs.uniform(0.1, 1, size=(16, 1)) + rs.randn(P + 1)).astype(np.float32)
    msgs = to_dev(K, X)[0]
    dst = torch.full((2, P + 1), NAN, device=K.dev)
    gam = torch.full((2, 1), NAN, device=K.dev)
    slots, honest = list(range(15)) + [-1], list(range(15))
    for rule in ("dnc", "gmed", "trim"):
        case = ("pipeline_std", rule, 3, slots, honest, P, "nnm")
        dst.fill_(NAN)
        K.ops.pipeline_attack([_job(K, dst[0], msgs, case, 2.0, gamma_out=gam[0])])
        _check(dst[0].cpu().numpy(), float(gam[0, 0]), X, case, 2.0, dict(exact=0, near=0, interior=0))
    # only DnC adds the fp64 mean: at 1422 parameters its job is one row of floats past the bound
    dst.fill_(NAN)
    gam.fill_(NAN)
    with pytest.raises(K.L.RcmarlError):
        K.ops.pipeline_attack([_job(K, dst[1], msgs, ("pipeline_std", "dnc", 3, slots, honest, P + 1, "nnm"), 2.0,
                                    gamma_out=gam[1])])
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(gam).all()
    assert np.array_equal(msgs.cpu().numpy(), X)


# ---------------------------------------------------------------------------------------------------------- Trainer
def _oracle_round(agents, labels, in_nodes, rows, attacks, rules, mixing, H, N, T, round_, seed, kernel_M, runs):
    """The oracle's round: the pipeline hook inside nnm_oracle's hook for the nnm receivers, inside the bucket hook for
    the bucketing receivers (the order of the Trainer's launches).  At a near tie of an attacker's mean objective the
    oracle follows the kernel's pick of that epoch (runs[e], a Trainer whose last epoch is e)."""
    gammas, objs = {}, {}
    inner = PA.make_hook(labels, in_nodes, attacks, rules, H, mixing, seed=seed, round_=round_, gammas=gammas,
                         objectives=objs, follow={e: r.attack_gammas() for e, r in enumerate(runs)})
    nnm = [m if m == "nnm" else None for m in mixing]
    if any(nnm):
        inner = NO.mixing_hook(labels, in_nodes, nnm, H, inner=inner, kernel_M=kernel_M)
    hook = BO.bucketing_hook(labels, in_nodes, mixing, seed, round_, inner=inner)
    loss = NO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=2, n_actor_steps=T, common_reward=False,
                           perm_source=NG._perms(), messages_hook=hook)
    return loss, gammas, objs


@pytest.mark.parametrize("rule,mixing", [("dnc", None), ("clip", "nnm"), ("trim", ("bucket", 2))])
def test_c2_update_round_with_a_pipeline_attacker(K, rule, mixing):
    """The benchmark's 5-agent team with agent 4 Byzantine on pipeline_std against receivers on `rule` after `mixing`
    (H = 1): two epochs against the oracle's round; one pipeline launch per epoch in place of the rcmarl_attack one;
    attack_gammas against the oracle's last epoch.  s = 1.5, so that no candidate is the min-max message itself
    (s = 2 makes candidate 16 exactly that message, which lies at the honest messages' largest distance: an exact
    boundary tie of the nnm selection inside the attacker's model, which fp32 and fp64 may break differently)."""
    w, desired, _ = pretrained()
    gamma, T, round_, N = 0.9, 40, 150, 64
    rs = np.random.RandomState(8600)
    rows = synth(rs, T * N)
    attack = ("pipeline_std", 1.5)
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule)
    mix = [mixing] * 4 + [None]
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mix if mixing else None)
    assert tr.pipe_pairs == [0, 1, 2] and tr.gamma_pairs == [0, 1, 2]
    agents = [NG._oracle_agent(rule, w[i], 0.01, gamma, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    NG._follow_dnc(agents, runs)
    want, gammas, objs = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: attack}, [rule] * 5, mix, [1] * 5, N, T,
                                       round_, 9, kernel_M, runs)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    TG._check_gammas(tr, gammas, objs)
    alie, _ = NG._trainer_round(dict(cfg, attack=("alie", 1.0)), rows, round_, 2, mix if mixing else None)
    assert tr.launches == alie.launches                     # one launch per epoch, pipeline or not


B16 = TG.B16
ATT16 = {1: ("pipeline_std", 2.0), 5: ("pipeline_std", 2.0), 9: ("pipeline_uv", 1.0), 11: ("alie", 1.0),
         14: ("pipeline_sgn", 2.0)}
RULES16 = ["dnc", "gmed", "trim", "scclip", "wmsr", "clip", "krum", "clip"]
MIX16 = ["nnm", ("bucket", 2), None, "nnm", ("bucket", 3), None, "nnm", None]


def test_16_agent_team_with_colluding_pipeline_attackers(K):
    """Circulant in-neighbourhoods of 10; four pipeline attackers (receivers hear several of them: colluding crafted
    slots) and one ALIE attacker, with Malicious and Greedy agents among the real slots; rules and mixing set per
    agent.  More than 32 pipeline jobs, so two launches per epoch."""
    from rcmarl import nets
    rs = np.random.RandomState(8700)
    NA = 16
    in_nodes = [[(i + k) % NA for k in range(10)] for i in range(NA)]
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    for i in range(NA):
        if B16[i] == "Malicious":
            w[i].append(nets.glorot_uniform(32, 1, rs))
    desired, fast = rs.randint(0, 10, size=(NA, 2)), [0.01 + 0.001 * (i % 4) for i in range(NA)]
    H = [1 + i % 2 for i in range(NA)]
    coop = [i for i, l in enumerate(B16) if l == "Cooperative"]
    rules, mixing = ["clip"] * NA, [None] * NA
    for q, i in enumerate(coop):
        rules[i], mixing[i] = RULES16[q], MIX16[q]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(B16):
        if lab == "Cooperative":
            agents.append(NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=B16, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma, H=H,
               fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4, aggregation=rules,
               attack=[ATT16.get(i) for i in range(16)])
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    assert 2 * len(tr.pipe_pairs) > 32 and tr.gamma_pairs == tr.pipe_pairs
    NG._follow_dnc(agents, runs)
    want, gammas, objs = _oracle_round(agents, B16, in_nodes, rows, ATT16, rules, mixing, H, N, T, round_, 4, kernel_M,
                                       runs)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({B16[i]}, {rules[i]}, {mixing[i]})")
    TG._check_gammas(tr, gammas, objs)


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


def test_world1_peer_comm_with_a_pipeline_attacker_is_bitwise(K, gloo_world1):
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["gmed", "dnc", "mkrum", "trim", "clip"], mixing=["nnm", "bucket", None, "nnm", None],
                     attack=("pipeline_std", 2.0))
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append(NG._state(tr) + [tr.att_gamma.clone()])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_train_rpbcac_with_a_pipeline_byzantine_agent(K):
    """Drop-in path: train_RPBCAC with Byzantine_CAC_agent(attack=("pipeline_uv", 2)) runs the same round as a Trainer
    built from the same objects with that attack passed directly, bit for bit."""
    import contextlib
    import io
    from agents.adversarial_CAC_agents import Byzantine_CAC_agent
    from rcmarl import api
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)

    def objects():
        env, agents, args = api.build_reference_objects(cfg)
        f = agents[4]
        agents[4] = Byzantine_CAC_agent(f.actor, f.critic, f.TR, 0.002, 0.9, attack=("pipeline_uv", 2))
        args["agent_label"] = C2_BYZ
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    env, agents, args = objects()
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(env, agents, args)
    tr = training.train_RPBCAC.last_trainer
    assert tr.pipe_pairs == [0, 1, 2] and tr.attack[4] == (K.L.PIPELINE_ATTACKS["pipeline_uv"], 2.0)
    direct = training.build_trainer(*objects())
    for _ in range(2):
        direct.rollout_block(4)
        direct.update_round()
    torch.cuda.synchronize()
    assert direct.launches == tr.launches
    for i in range(5):
        for a, b in zip(tr.get_weights(i), direct.get_weights(i)):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
    assert all(np.isfinite(g).all() for g in tr.attack_gammas().values())
