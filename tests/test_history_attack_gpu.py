"""GPU parity of the momentum-aware Byzantine messages (rcmarl_history_attack, include/rcmarl.h): at c = 0 and
first = 1 bitwise rcmarl_pipeline_attack without mixing (M, not read, NaN) for every rule at n_in 2..16; model_out
bitwise the receiver's real chain (rcmarl_momentum_mix on a copy of M, then rcmarl_consensus_hidden /
rcmarl_vector_aggregate / rcmarl_dnc_aggregate) with every crafted message sent, with and without colluders, over every
family x rule, beta 0 / 0.5 / 0.9 / 0.99 x first 0 / 1, repeated real slots, Malicious-style real slots and +-inf /
1e30 in messages and in M, up to 1421 parameters at n_in 16 under DnC at the staging bound; momentum and ref bitwise
untouched; the pick and the message against the fp64 oracle (tests/history_attack_oracle.py); bitwise determinism across job orders and launch
splits; the refusals; and whole update rounds through Trainer -- C2 with agent 4 on history_* against receivers on
momentum before clip, dnc and gmed against the fp64 oracle, a 16-agent team with five colluding history attackers
beside momentum and plain receivers (two history launches and a pipeline launch per epoch) against the fp64 oracle,
and history_* against receivers without momentum bitwise pipeline_*.

Near ties are handled as in test_pipeline_attack_gpu.py: where the oracle's relative margin between its best and its
second-best distinct objective exceeds MARGIN = 1e-4 the kernel's pick must be the oracle's, and otherwise the fp64
objective of the kernel's pick must lie within MARGIN relative of the maximum; in whole rounds the oracle's attacker
follows the kernel's pick at such a near tie."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import history_attack_oracle as HO                      # noqa: E402
import team_util as TU                                  # noqa: E402
import test_nnm_gpu as NG                               # noqa: E402  (the C2 round helpers)
from golden_util import pretrained                      # noqa: E402
from kernel_util import close, load_kernels, synth      # noqa: E402
from oracle import rpbcac_oracle as O                   # noqa: E402  (checker only)

f32, f64 = np.float32, np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
MARGIN = 1e-4
N_REAL, S = 20, 1427                                    # real message rows (16 .. 19 Malicious-style) and the stride
RULES = ("clip", "trim", "wmsr", "krum", "mkrum", "scclip", "gmed", "dnc")
BETAS = (0.0, 0.5, 0.9, 0.99)


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _max_h(rule, n):
    if rule in ("krum", "mkrum"):
        return n - 3
    if rule == "trim":
        return (n - 1) // 2
    return n - 1


def _cases(rs, colluders):
    """(rule, H, slots, honest, own, P, beta, first) for every rule x beta x first at n_in 2..16: 1-3 crafted slots, all
    own (one attacker, repeats allowed) or, with colluders, one attacker per crafted slot; in every other case some real
    message sits in two slots (each slot keeps its own state, so the two give different momentum rows); P among the
    trainer's parameter counts."""
    out = []
    t = 0
    for n_in in range(2, 17):
        for rule in RULES:
            if rule in ("krum", "mkrum") and n_in < 3:
                continue
            n_cr = 1 + rs.randint(min(3, n_in - 1))
            if colluders and n_in > 2:
                n_cr = max(n_cr, 2)
            real = [int(x) for x in rs.choice(N_REAL, size=n_in - n_cr, replace=False)]
            if real[0] >= 16:                                             # the own slot is honest
                real[0] = int(rs.choice([r for r in range(16) if r not in real[1:]]))
            if t % 2 and len(real) >= 3:                                  # a repeated real slot
                real[-1] = real[int(rs.randint(len(real) - 1))]
            slots = real[:1] + [-1] * n_cr + real[1:]
            rest = slots[1:]
            rs.shuffle(rest)
            slots[1:] = rest
            honest = [k for k, s in enumerate(slots) if 0 <= s < 16]
            crafted = [k for k, s in enumerate(slots) if s < 0]
            own = crafted[:1] if colluders else crafted
            H = min(int(rs.randint(0, 3)), max(_max_h(rule, n_in), 0))
            P = int(rs.choice([1, 33, 200, 661, 761, 1101]))
            out.append((rule, H, slots, honest, own, P, BETAS[t % 4], (t // 4) % 2))
            t += 1
    return out


class Buffers:
    """The message stack (N_REAL real rows, then one row per attacker), and per job a ref, n_in M rows at stride S and
    dst / gamma / model_out rows, all pre-filled with NaN; row 16.. of the stack carries +-inf / 1e30 when poisoned."""

    def __init__(self, K, rs, n_jobs, poison=False):
        self.K = K
        centre = rs.randn(S)
        stack = (centre + rs.randn(N_REAL, S) * rs.uniform(0.05, 1.0, size=(N_REAL, 1))).astype(f32)
        stack[16:] += (rs.randn(4, S) * 3.0).astype(f32)
        if poison:
            stack[17, ::5] = np.inf
            stack[18] = 1e30
            stack[19, 1::7] = -np.inf
        self.stack = stack
        self.msgs = torch.full((N_REAL + 16, S), NAN, device=K.dev)
        self.msgs[:N_REAL] = torch.as_tensor(stack).to(K.dev)
        self.ref = torch.as_tensor((centre + rs.randn(n_jobs, S) * 0.2).astype(f32)).to(K.dev)
        M = (rs.randn(n_jobs, 16, S) * 0.3).astype(f32)
        if poison:
            M[:, 3, ::11] = np.inf
            M[:, 5, 2::9] = -np.inf
            M[:, 6, ::4] = 1e30
        self.M = torch.as_tensor(M).to(K.dev)
        self.dst = torch.full((n_jobs, S), NAN, device=K.dev)
        self.gam = torch.full((n_jobs, 2), NAN, device=K.dev)
        self.model = torch.full((n_jobs, S), NAN, device=K.dev)

    def job(self, j, case, scale=2.0, attack="history_std", own=None, dst=None, ref=None, M=None, first=None):
        rule, H, slots, honest, own0, P, beta, first0 = case
        return self.K.ops.history_attack_job(
            self.dst[j] if dst is None else dst, self.msgs, S, P, slots, honest, rule, H, attack, scale,
            self.ref[j] if ref is None else ref, self.M[j] if M is None else M, S, beta,
            first0 if first is None else first, own0 if own is None else own, gamma_out=self.gam[j, :1],
            model_out=self.model[j])


def _rule_out(K, stack, nodes, P, rule, H):
    out = torch.full((S,), NAN, device=K.dev)
    if rule == "dnc":
        K.ops.dnc_aggregate([K.ops.vector_job(out, stack, S, P, nodes, H, K.L.SPECTRAL_DNC)])
    elif rule in ("krum", "mkrum", "scclip", "gmed"):
        K.ops.vector_aggregate([K.ops.vector_job(out, stack, S, P, nodes, H, rule)])
    else:
        K.ops.consensus_hidden([K.ops.consensus_job(out, stack, S, P, nodes, H, rule)])
    return out


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def _receiver(K, B, j, case, sent):
    """The receiver's real chain: rcmarl_momentum_mix of the slots (crafted slot k receiving the stack row sent[k]) on a
    copy of M, then its rule; returns the aggregate [S]."""
    rule, H, slots, honest, own, P, beta, first = case
    nodes = [sent[k] if s < 0 else s for k, s in enumerate(slots)]
    rows = torch.full((len(slots), S), NAN, device=K.dev)
    M = B.M[j].clone()
    K.ops.momentum_mix([K.ops.momentum_job(rows, B.msgs, S, P, nodes, B.ref[j], M, S, beta, first)])
    return _rule_out(K, rows, list(range(len(slots))), P, rule, H)


def test_at_c_zero_and_first_step_bitwise_the_pipeline_attack(K):
    """Every rule x direction at n_in 2..16: dst, gamma_out and model_out bit for bit; M (NaN) is not read."""
    rs = np.random.RandomState(9500)
    cases = _cases(rs, False)
    B = Buffers(K, rs, 32)
    B.ref.zero_()
    B.M.fill_(NAN)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        for d in ("uv", "std", "sgn"):
            B.dst.fill_(NAN), B.gam.fill_(NAN), B.model.fill_(NAN)
            K.ops.history_attack([B.job(j, c, attack="history_" + d, first=1) for j, c in enumerate(part)])
            pdst, pgam, pmod = (torch.full_like(x, NAN) for x in (B.dst, B.gam, B.model))
            K.ops.pipeline_attack([K.ops.pipeline_attack_job(pdst[j], B.msgs, S, P, slots, hon, rule, H,
                                                             "pipeline_" + d, 2.0, gamma_out=pgam[j, :1],
                                                             model_out=pmod[j])
                                   for j, (rule, H, slots, hon, _, P, _, _) in enumerate(part)])
            torch.cuda.synchronize()
            for x, y in ((B.dst, pdst), (B.gam, pgam), (B.model, pmod)):
                assert np.array_equal(_bits(x[:len(part)]), _bits(y[:len(part)])), d


@pytest.mark.parametrize("colluders", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_model_out_is_what_the_receiver_computes(K, colluders, poison):
    """Every crafted message sent (each colluder runs its own job with the same parameters): rcmarl_momentum_mix on a
    copy of M, then the rule, equals model_out bit for bit; momentum and ref are untouched."""
    rs = np.random.RandomState(9600 + 2 * colluders + poison)
    cases = _cases(rs, colluders)
    assert {c[0] for c in cases} == set(RULES) and {(c[6], c[7]) for c in cases} == {(b, f) for b in BETAS
                                                                                      for f in (0, 1)}
    assert sum(len({x for x in c[2] if x >= 0}) < sum(x >= 0 for x in c[2]) for c in cases) > len(cases) // 4
    B = Buffers(K, rs, len(cases), poison)
    for q, case in enumerate(cases):                   # poison only the M rows of slots outside the honest set
        B.M[q, case[3]] = torch.as_tensor((rs.randn(len(case[3]), S) * 0.3).astype(f32)).to(K.dev)
    M0, ref0 = B.M.clone(), B.ref.clone()
    n_att = 0
    for q, case in enumerate(cases):
        # one launch per receiver: attacker i writes stack row N_REAL + i, its model_out row q * 3 + i mod 32
        crafted = [k for k, s in enumerate(case[2]) if s < 0]
        groups = [[k] for k in crafted] if colluders else [crafted]
        B.msgs[N_REAL:].fill_(NAN)
        B.model.fill_(NAN)
        jobs, sent = [], {}
        for i, grp in enumerate(groups):
            j = K.ops.history_attack_job(B.msgs[N_REAL + i], B.msgs, S, case[5], case[2], case[3], case[0], case[1],
                                         "history_std", 2.0, B.ref[q], B.M[q], S, case[6], case[7], grp,
                                         model_out=B.model[i])
            jobs.append(j)
            sent.update({k: N_REAL + i for k in grp})
        K.ops.history_attack(jobs)
        torch.cuda.synchronize()
        want = _receiver(K, B, q, case, sent)
        P = case[5]
        for i in range(len(groups)):
            assert np.array_equal(_bits(B.model[i, :P]), _bits(want[:P])), (case, colluders, poison)
            assert torch.isnan(B.model[i, P:]).all() and torch.isnan(B.msgs[N_REAL + i, P:]).all()
            n_att += 1
    assert torch.equal(B.M.nan_to_num(7.0), M0.nan_to_num(7.0)) and torch.equal(B.ref, ref0)
    assert n_att >= len(cases)


def test_pick_and_message_against_the_oracle(K):
    """The pick against the fp64 oracle (on the fp32 inputs) with the margin rule, and the crafted row against the
    target: one momentum step of dst (momentum_oracle.step, the receiver's arithmetic) lands on m(gamma_i*)."""
    rs = np.random.RandomState(9700)
    cases = _cases(rs, True)[::2]
    B = Buffers(K, rs, 32)
    stats = dict(exact=0, near=0, interior=0)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        B.dst.fill_(NAN), B.gam.fill_(NAN)
        K.ops.history_attack([B.job(j, c) for j, c in enumerate(part)])
        dst, gam = B.dst.cpu().numpy(), B.gam.cpu().numpy()
        ref, M = B.ref.cpu().numpy(), B.M.cpu().numpy()
        for j, (rule, H, slots, honest, own, P, beta, first) in enumerate(part):
            tag = f"{rule} H={H} slots={slots} own={own} P={P} beta={beta} first={first}"
            rows = B.stack[:, :P].astype(f64)
            m, g, Ob, R, Y = HO.craft(rows, slots, honest, rule, H, "history_std", 2.0, ref[j, :P].astype(f64),
                                      M[j, :, :P].astype(f64), beta, bool(first), own)
            gg = float(gam[j, 0])
            mu, d, g_mm = HO.AA.gamma_of(Y[honest], "minmax_std")
            G = 2.0 * float(g_mm)
            i_gpu = 0 if G == 0 else int(round(gg / G * HO.STEPS))
            if G != 0:
                close(gg, G * i_gpu / HO.STEPS, rtol=1e-3, atol=0, err_msg=tag)
            top, i_or = Ob.max(), int(np.argmax(Ob))
            if not np.isfinite(top):
                assert i_gpu == 0, tag
                continue
            if HO.TA.margin(Ob) > MARGIN:
                assert i_gpu == i_or, f"{tag}: picked {i_gpu}, oracle {i_or}"
                stats["exact"] += 1
            else:
                assert Ob[i_gpu] >= top - MARGIN * abs(top), tag
                stats["near"] += 1
            stats["interior"] += 0 < i_gpu < HO.STEPS
            k0 = min(own)
            row = HO.step_row(dst[j, :P], ref[j, :P], M[j, k0, :P], beta, bool(first))
            t = HO.TA.candidate(mu, d, f64(gg))
            close(row, t, rtol=2e-3, atol=2e-3 * max(1.0, float(np.abs(t).max())), err_msg=tag)
    print(stats)
    assert stats["exact"] > len(cases) // 2 and stats["interior"] > 0


def test_staging_bound_1421_parameters_at_n_in_16_under_dnc(K):
    rs = np.random.RandomState(9800)
    B = Buffers(K, rs, 1)
    case = ("dnc", 3, list(range(15)) + [-1], list(range(15)), [15], 1421, 0.9, 0)
    K.ops.history_attack([B.job(0, case, dst=B.msgs[N_REAL], M=B.M[0], ref=B.ref[0])])
    want = _receiver(K, B, 0, case, {15: N_REAL})
    assert np.array_equal(_bits(B.model[0, :1421]), _bits(want[:1421]))
    assert torch.isfinite(B.msgs[N_REAL, :1421]).all() and float(B.gam[0, 0]) > 0


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(9900)
    cases = _cases(rs, True)[::4][:32]
    B = Buffers(K, rs, 32)

    def run(groups):
        for x in (B.dst, B.gam, B.model):
            x.fill_(NAN)
        for g in groups:
            K.ops.history_attack([B.job(j, cases[j]) for j in g])
        return [torch.nan_to_num(x, 7.0).clone() for x in (B.dst, B.gam, B.model)]
    every = list(range(len(cases)))
    first = run([every])
    for groups in ([every], [every[::-1]], [every[5:9], every[:5], every[9:]], [[j] for j in every]):
        assert all(torch.equal(a, b) for a, b in zip(run(groups), first))


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(10000)
    B = Buffers(K, rs, 4)
    case = ("clip", 1, [0, 1, -1, 3], [0, 1, 3], [2], 300, 0.9, 0)
    good = B.job(0, case)
    J = lambda **kw: B.job(1, case, **kw)                               # noqa: E731
    bad = [J(own=[]), J(own=[1]), J(own=[0]),                           # no own slot, own bits on real slots
           J(dst=B.msgs[1]), J(dst=B.ref[0]), J(dst=B.M[1, 3]),         # dst on a slot row, a ref, an M row
           J(ref=B.dst[0]), J(M=B.model[0:1]),                          # ref / M rows on the other job's outputs
           J(first=2), J(dst=B.dst[0])]                                 # first not 0 / 1, dsts that overlap
    j = B.job(1, case)
    j.beta = 1.0
    bad.append(j)
    j = B.job(1, case)
    j.attack.family, j.attack.rule = 2, 1                                # SPECTRAL with a rule other than DnC
    bad.append(j)
    snap = [x.clone() for x in (B.msgs, B.ref, B.M)]
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.history_attack([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(B.dst).all() and torch.isnan(B.gam).all() and torch.isnan(B.model).all()
    for a, b in zip(snap, (B.msgs, B.ref, B.M)):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))
    K.ops.history_attack([good])
    assert torch.isfinite(B.dst[0, :300]).all() and torch.isnan(B.dst[1]).all()


# ---------------------------------------------------------------------------------------------------------- Trainer
def _cfg(rule, attack):
    w, desired, _ = pretrained()
    return dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1, fast_lr=0.01,
                slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule)


@pytest.mark.parametrize("rule,beta,name", [("clip", 0.9, "history_std"), ("dnc", 0.99, "history_uv"),
                                            ("gmed", 0.9, "history_sgn")])
def test_c2_update_round_against_the_oracle(K, rule, beta, name):
    """C2 with agent 4 on `name` (s = 2) and every cooperative agent on momentum `beta` before `rule` (H = 1): one
    update round of two epochs against the fp64 oracle, the attack reading M before each epoch's momentum step; one
    history launch per epoch, as
    many launches as with the gauss attack."""
    cfg = _cfg(rule, (name, 2.0))
    rs = np.random.RandomState(10100)
    T, N, round_ = 40, 64, 150
    rows = synth(rs, T * N)
    tr, got, _, runs = NG._kernel_M(dict(cfg, momentum=beta), rows, round_, None)
    assert tr.hist_pairs == [0, 1, 2] and tr.pipe_pairs == [] and tr.momentum_steps == [2] * 4
    w = cfg["weights"]
    agents = [NG._oracle_agent(rule, w[i], 0.01, 0.9, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, 0.9, dtype=f64))
    NG._follow_dnc(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = HO.momentum_hook(agents, C2_BYZ, IN_NODES, {4: (name, 2.0)}, [rule] * 5, 1, [beta] * 4 + [None], seed=9,
                            round_=round_, follow=follow, gammas=gammas)
    want = HO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                           common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    kg = tr.attack_gammas()
    for key, g in gammas.items():
        close(kg[key], np.asarray(g, f32), rtol=2e-3, atol=1e-6, err_msg=str(key))
    plain, _ = NG._trainer_round(dict(cfg, attack=("gauss", 1.0), momentum=beta), rows, round_, 2, None)
    assert tr.launches == plain.launches                                        # one attack launch per epoch


RULES16 = ["clip", "dnc", "trim", "wmsr", "scclip", "gmed", "mkrum", "clip"]   # the 8 cooperative agents, in order
MOM16 = [0.9, 0.99, 0.5, None, 0.9, 0.9, 0.99, 0.9]                             # receiver 6 without momentum
HIST16 = {1: ("history_std", 2.0), 5: ("history_uv", 2.0), 9: ("history_sgn", 1.5), 11: ("history_std", 1.0),
          14: ("history_uv", 0.5)}


def test_16_agent_team_with_colluding_history_attackers(K):
    """16 agents (8 cooperative, 5 Byzantine all on history_*, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, receiver
    0 listing attacker 1 twice): 7 receivers on momentum hear 2-3 colluding history attackers each (17 pairs, 34 jobs,
    two history launches per epoch), receiver 6 without momentum gets the pipeline jobs of its 2 pairs.  One update
    round of two epochs against the fp64 oracle through history_attack_oracle.momentum_hook: losses, weights and every
    pair's gamma."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, _ = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mom = ["clip"] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mom[i] = RULES16[q], MOM16[q]
    H = [max(h, 1) if rules[i] == "dnc" else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[HIST16.get(i) for i in range(16)], momentum=mom)
    tr, got, _, runs = NG._kernel_M(cfg, rows, round_, None)
    hist_mom = [e for e in tr.hist_pairs if mom[tr.byz_pairs[e][1]] is not None]
    assert len(tr.hist_pairs) == 19 and len(hist_mom) == 17 and tr.pipe_pairs == []
    assert sorted({tr.byz_pairs[e][1] for e in tr.hist_pairs if e not in hist_mom}) == [6]
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    NG._follow_dnc(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = HO.momentum_hook(agents, labels, in_nodes, HIST16, rules, H, mom, seed=4, round_=round_, follow=follow,
                            gammas=gammas)
    want = HO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                           common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]}, {mom[i]})")
    kg = tr.attack_gammas()
    assert sorted(kg) == sorted(gammas) and len(kg) == 19
    for key, g in gammas.items():
        close(kg[key], np.asarray(g, f32), rtol=2e-3, atol=1e-6, err_msg=str(key))
    plain, _ = NG._trainer_round(dict(cfg, attack=[("gauss", 0.5) if i in HIST16 else None for i in range(16)]), rows,
                                 round_, 2, None)
    # per epoch two history launches (32 + 2 jobs) and one pipeline launch, against gauss's two attack launches
    assert tr.launches - plain.launches == 2


@pytest.mark.parametrize("rule,mixing", [("clip", None), ("dnc", None), ("trim", "nnm"), ("gmed", ("bucket", 2))])
def test_without_momentum_history_is_the_pipeline_attack_bitwise(K, rule, mixing):
    cfg = _cfg(rule, None)
    rs = np.random.RandomState(10200)
    rows = synth(rs, 40 * 64)
    out = {}
    for name in ("history_uv", "pipeline_uv"):
        tr, got = NG._trainer_round(dict(cfg, attack=(name, 2.0)), rows, 150, 2, mixing)
        out[name] = (tr.msg_c[5:8].clone(), tr.msg_t[5:8].clone(), tr.attack_gammas(), tr.critic.clone(), tr.launches)
    a, b = out["history_uv"], out["pipeline_uv"]
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3]) and a[4] == b[4]
    assert {k: v.tolist() for k, v in a[2].items()} == {k: v.tolist() for k, v in b[2].items()}
