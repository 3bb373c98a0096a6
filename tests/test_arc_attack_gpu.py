"""GPU parity of the ARC-aware Byzantine messages (rcmarl_pipeline_arc_attack, rcmarl_history_arc_attack,
include/rcmarl.h): at H = 0 bitwise the base attacks for every rule x direction x mixing; model_out bitwise the
receiver's real chain ([rcmarl_momentum_mix on a copy of M] -> rcmarl_arc_clip -> [rcmarl_nnm_mix] -> the rule) with
every crafted message sent, with and without colluders and with poisoned non-honest slots; under bucketing sample 0
against the fp32 oracle; the pick against the fp64 oracle (tests/arc_attack_oracle.py) with the margin rule of
test_pipeline_attack_gpu.py; bitwise determinism across job orders and launch splits; the refusals; and whole update
rounds through Trainer -- C2 with agent 4 on arc_std against receivers that clip before seven pipelines, a 16-agent team
with colluding arc_* attackers, and train_RPBCAC with an arc_* Byzantine agent."""
import contextlib
import io

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import arc_attack_oracle as AAO                         # noqa: E402
import arc_oracle as AO                                 # noqa: E402
import bucket_oracle as BO                              # noqa: E402
import pipeline_attack_oracle as PA                     # noqa: E402
import team_util as TU                                  # noqa: E402
import test_arc_gpu as AG                               # noqa: E402  (the C2 oracle agents)
import test_history_attack_gpu as HG                    # noqa: E402  (the history buffers and cases)
import test_nnm_gpu as NG                               # noqa: E402  (the C2 round helpers)
import test_pipeline_attack_gpu as PG                   # noqa: E402  (the pipeline cases)
import test_tailored_attacks_gpu as TG                  # noqa: E402  (the message stacks)
from golden_util import pretrained                      # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                   # noqa: E402  (checker only)

f32, f64 = np.float32, np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
MARGIN = 1e-4
WORDS = PG.WORDS


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def _arc_h(rule, n_rows, n_in, rs):
    """An H in 1..3 that the rule admits at n_rows (ARC's own bound, H < n_in, follows)."""
    return max(1, min(int(rs.randint(1, 4)), PG._max_h(rule, n_rows), n_in - 1))


def _pipe_cases(rs, n_rows, mixings=(None, "nnm"), colluders=False):
    """(attack, rule, H, slots, honest, P, mixing) with n_in 4..16, slot 0 real and honest, H 1..3, 1-3 crafted slots."""
    out = []
    t = 0
    for n_in in range(4, 17):
        for rule in PA.RULES:
            mixing = mixings[t % len(mixings)]
            n_cr = 1 + rs.randint(min(3, n_in - 2)) if not colluders else 2 + rs.randint(2)
            real = [int(x) for x in rs.choice(n_rows, size=n_in - n_cr, replace=False)]
            if real[0] >= n_rows - 4:
                real[0] = int(rs.choice([r for r in range(n_rows - 4) if r not in real[1:]]))
            slots = real[:1] + [-1] * n_cr + real[1:]
            rest = slots[1:]
            rs.shuffle(rest)
            slots[1:] = rest
            honest = [k for k, s in enumerate(slots) if 0 <= s < n_rows - 4]
            nr = PA.n_rows(n_in, mixing)
            if (rule in ("krum", "mkrum") and nr < 4) or PG._max_h(rule, nr) < 1:
                continue
            H = _arc_h(rule, nr, n_in, rs)
            P = int(rs.choice([33, 200, 661, 761]))
            out.append(("arc_" + AAO.AA.DEVS[t % 3], rule, H, slots, honest, P, mixing))
            t += 1
    return out


def _pjob(K, dst, msgs, case, gamma_out=None, model_out=None, scale=2.0, n_perms=3):
    return PG._job(K, dst, msgs, case, scale, gamma_out=gamma_out, model_out=model_out, n_perms=n_perms)


def _pipe_chain(K, msgs, stride, case, sent_row):
    """The receiver's chain on the stack with every crafted slot reading row sent_row: rcmarl_arc_clip, then
    rcmarl_nnm_mix if it mixes, then its rule."""
    attack, rule, H, slots, honest, P, mixing = case
    nodes = [sent_row if s < 0 else s for s in slots]
    clipped = torch.full((len(slots), stride), NAN, device=K.dev)
    K.ops.arc_clip([K.ops.vector_job(clipped, msgs, stride, P, nodes, H, K.L.MIX_ARC)])
    stack, nodes = clipped, list(range(len(slots)))
    if mixing == "nnm":
        mixed = torch.full((len(slots), stride), NAN, device=K.dev)
        K.ops.nnm_mix([K.ops.vector_job(mixed, stack, stride, P, nodes, H, K.L.MIX_NNM)])
        stack = mixed
    out = torch.full((stride,), NAN, device=K.dev)
    if rule == "dnc":
        K.ops.dnc_aggregate([K.ops.vector_job(out, stack, stride, P, nodes, H, K.L.SPECTRAL_DNC)])
    elif rule in ("krum", "mkrum", "scclip", "gmed"):
        K.ops.vector_aggregate([K.ops.vector_job(out, stack, stride, P, nodes, H, rule)])
    else:
        K.ops.consensus_hidden([K.ops.consensus_job(out, stack, stride, P, nodes, H, rule)])
    return out


def _hist_chain(K, B, j, case, sent):
    """The history form's receiver chain: rcmarl_momentum_mix on a copy of M, rcmarl_arc_clip, then the rule."""
    rule, H, slots, honest, own, P, beta, first = case
    nodes = [sent[k] if s < 0 else s for k, s in enumerate(slots)]
    rows = torch.full((len(slots), HG.S), NAN, device=K.dev)
    M = B.M[j].clone()
    K.ops.momentum_mix([K.ops.momentum_job(rows, B.msgs, HG.S, P, nodes, B.ref[j], M, HG.S, beta, first)])
    clipped = torch.full_like(rows, NAN)
    K.ops.arc_clip([K.ops.vector_job(clipped, rows, HG.S, P, list(range(len(slots))), H, K.L.MIX_ARC)])
    return HG._rule_out(K, clipped, list(range(len(slots))), P, rule, H)


# --------------------------------------------------------------------------------------------------- 1. H = 0
def test_at_h0_pipeline_form_is_bitwise_the_pipeline_attack(K):
    """Every rule x direction x mixing at n_in 2..16 with finite inputs (k_clip = 0): dst, gamma_out and model_out."""
    rs = np.random.RandomState(11100)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = [(a, r, 0, s, h, P, m) for (a, r, H, s, h, P, m) in PG._cases(rs, stack.shape[0]) if s[0] >= 0]
    assert {c[1] for c in cases} == set(PA.RULES) and {str(c[6]) for c in cases} == {str(m) for m in PG.MIXINGS}
    assert {c[0] for c in cases} == set(PA.ATTACKS)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        out = []
        for launch in (K.ops.pipeline_attack, K.ops.pipeline_arc_attack):
            dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
            gam = torch.full((len(part), 1), NAN, device=K.dev)
            model = torch.full_like(dst, NAN)
            launch([_pjob(K, dst[j], msgs, c, gamma_out=gam[j], model_out=model[j]) for j, c in enumerate(part)])
            out.append((dst, gam, model))
        torch.cuda.synchronize()
        for x, y in zip(*out):
            assert np.array_equal(_bits(x), _bits(y))


def test_at_h0_history_form_is_bitwise_the_history_attack(K):
    rs = np.random.RandomState(11200)
    cases = [c[:1] + (0,) + c[2:] for c in HG._cases(rs, True)]
    assert {c[0] for c in cases} == set(HG.RULES)
    B = HG.Buffers(K, rs, 32)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        for d in ("uv", "std", "sgn"):
            out = []
            for launch, name in ((K.ops.history_attack, "history_" + d), (K.ops.history_arc_attack, "arc_" + d)):
                B.dst.fill_(NAN), B.gam.fill_(NAN), B.model.fill_(NAN)
                launch([B.job(j, c, attack=name) for j, c in enumerate(part)])
                out.append([x.clone() for x in (B.dst, B.gam, B.model)])
            torch.cuda.synchronize()
            for x, y in zip(*out):
                assert np.array_equal(_bits(x), _bits(y)), d


# ----------------------------------------------------------------------------------------- 2. model_out = the chain
def _poisoned_stack(rs, poison):
    stack = TG._stack(rs)
    if poison:                                          # rows outside every honest set (the last 4)
        stack[-4, ::5] = np.inf
        stack[-3] = 1e30
        stack[-2, 1::7] = -np.inf
    return stack


@pytest.mark.parametrize("colluders", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_pipeline_form_model_out_is_what_the_receiver_computes(K, colluders, poison):
    rs = np.random.RandomState(11300 + 2 * colluders + poison)
    stack = _poisoned_stack(rs, poison)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    cases = _pipe_cases(rs, n_rows, colluders=colluders)
    assert {c[1] for c in cases} == set(PA.RULES) and {c[2] for c in cases} == {1, 2, 3}
    for case in cases:
        model = torch.full((stride,), NAN, device=K.dev)
        msgs[n_rows].fill_(NAN)
        K.ops.pipeline_arc_attack([_pjob(K, msgs[n_rows], msgs, case, model_out=model)])
        want = _pipe_chain(K, msgs, stride, case, n_rows)
        torch.cuda.synchronize()
        P = case[5]
        assert np.array_equal(_bits(model[:P]), _bits(want[:P])), case
        assert torch.isnan(model[P:]).all()


@pytest.mark.parametrize("colluders", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_history_form_model_out_is_what_the_receiver_computes(K, colluders, poison):
    rs = np.random.RandomState(11400 + 2 * colluders + poison)
    cases = []
    for t, c in enumerate(HG._cases(rs, colluders)):
        rule, H, slots, honest, own, P, beta, first = c
        if len(slots) < 4 or (rule in ("krum", "mkrum") and len(slots) < 5):
            continue
        H = max(1, min(1 + t % 3, HG._max_h(rule, len(slots))))
        cases.append((rule, H, slots, honest, own, P, (0.0, 0.9)[t % 2], (t // 2) % 2))
    assert {c[1] for c in cases} == {1, 2, 3} and {(c[6], c[7]) for c in cases} == {(b, f) for b in (0.0, 0.9)
                                                                                      for f in (0, 1)}
    B = HG.Buffers(K, rs, len(cases), poison)
    for q, case in enumerate(cases):                   # poison only the M rows of slots outside the honest set
        B.M[q, case[3]] = torch.as_tensor((rs.randn(len(case[3]), HG.S) * 0.3).astype(f32)).to(K.dev)
    M0, ref0 = B.M.clone(), B.ref.clone()
    for q, case in enumerate(cases):
        crafted = [k for k, s in enumerate(case[2]) if s < 0]
        groups = [[k] for k in crafted] if colluders else [crafted]
        B.msgs[HG.N_REAL:].fill_(NAN)
        B.model.fill_(NAN)
        jobs, sent = [], {}
        for i, grp in enumerate(groups):
            jobs.append(K.ops.history_attack_job(B.msgs[HG.N_REAL + i], B.msgs, HG.S, case[5], case[2], case[3],
                                                 case[0], case[1], "arc_std", 2.0, B.ref[q], B.M[q], HG.S, case[6],
                                                 case[7], grp, model_out=B.model[i]))
            sent.update({k: HG.N_REAL + i for k in grp})
        K.ops.history_arc_attack(jobs)
        want = _hist_chain(K, B, q, case, sent)
        torch.cuda.synchronize()
        P = case[5]
        for i in range(len(groups)):
            assert np.array_equal(_bits(B.model[i, :P]), _bits(want[:P])), (case, colluders, poison)
    assert torch.equal(B.M.nan_to_num(7.0), M0.nan_to_num(7.0)) and torch.equal(B.ref, ref0)


def test_pipeline_form_under_bucketing_model_out_is_sample_zero(K):
    """rcmarl_arc_clip on the slots with the crafted message, then sample 0's buckets and the rule in the fp32 oracle."""
    rs = np.random.RandomState(11500)
    stack = TG._stack(rs, n_bad=0)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    cases = [c for c in _pipe_cases(rs, n_rows, mixings=(("bucket", 2), ("bucket", 3)))
             if c[1] in ("clip", "trim", "wmsr")][:24]
    for case in cases:
        attack, rule, H, slots, honest, P, mixing = case
        model = torch.full((stride,), NAN, device=K.dev)
        K.ops.pipeline_arc_attack([_pjob(K, msgs[n_rows], msgs, case, model_out=model)])
        clipped = torch.full((len(slots), stride), NAN, device=K.dev)
        K.ops.arc_clip([K.ops.vector_job(clipped, msgs, stride, P, [n_rows if s < 0 else s for s in slots], H,
                                         K.L.MIX_ARC)])
        Y = clipped[:, :P].cpu().numpy()
        bks = PA.buckets(len(slots), mixing[1], WORDS["seed"], 0,
                         *[WORDS[k] for k in ("attacker", "receiver", "net", "round_", "epoch")])
        want = PA.rule_output(BO.mix(Y, bks)[0], rule, H)
        close(model[:P].cpu().numpy(), want, rtol=1e-5, atol=1e-6, err_msg=str(case))


# ------------------------------------------------------------------------------------------- 3. the pick vs fp64
def _near_tie(rows, slots, honest, attack, g, H, mixing, rel=1e-4):
    """Whether fp32 may order the candidate's clipped slot list differently from fp64: ARC's d_k at tau's rank, or,
    under nnm, a row's n_in - H nearest clipped rows, within `rel` of the next.  ARC makes such ties exact: a clipped row
    lies at tau from x_0, as the row that set tau does."""
    V = np.stack([rows[slots[k]] for k in honest])
    mu, d, _ = AAO.AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    X = np.stack([AAO.TA.candidate(mu, d, g) if s < 0 else rows[s] for s in slots])
    n, kc = len(slots), AO.k_clip(H, len(slots))
    ds = np.sort(AO.distances(X)[1:])[::-1]

    def close_pair(a, b):
        return np.isfinite(a) and np.isfinite(b) and abs(a - b) <= rel * max(abs(a), abs(b), 1e-30)
    if kc < n - 1 and any(close_pair(ds[i], ds[i + 1]) for i in range(max(kc - 1, 0), min(kc + 1, n - 2))):
        return True
    if mixing == "nnm":
        Y = AO.clip(X, H)[0]
        D = np.sqrt(((Y[:, None] - Y[None]) ** 2).sum(-1))
        m = n - H
        for k in range(n):
            s = np.sort(D[k])
            if m < n and close_pair(s[m - 1], s[m]):
                return True
    return False


def test_pick_against_the_oracle(K):
    """The pipeline form's pick against the fp64 oracle with the margin rule, except where the candidates the two
    picks name sit at a near tie of the clipping or nnm order (_near_tie).  Among the cases there are interior picks,
    picks whose crafted row ARC clips (0 < c < 1), and picks that differ from pipeline_*'s on the same inputs."""
    rs = np.random.RandomState(11600)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    n_rows, stride = stack.shape
    cases = _pipe_cases(rs, n_rows, mixings=(None, "nnm", ("bucket", 2)))[::2]
    stats = dict(exact=0, near=0, tie=0, interior=0, clipped=0, differs=0)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        gams = []
        for launch, pre in ((K.ops.pipeline_arc_attack, "arc_"), (K.ops.pipeline_attack, "pipeline_")):
            dst = torch.full((len(part), stride), NAN, device=K.dev)
            gam = torch.full((len(part), 1), NAN, device=K.dev)
            launch([_pjob(K, dst[j], msgs, (pre + c[0].split("_")[1],) + c[1:], gamma_out=gam[j])
                    for j, c in enumerate(part)])
            gams.append(gam.cpu().numpy()[:, 0])
        for j, (attack, rule, H, slots, honest, P, mixing) in enumerate(part):
            tag = f"{attack} {rule} H={H} {mixing} slots={slots} P={P}"
            rows = stack[:, :P].astype(f64)
            _, _, Ob, _, c = AAO.craft_pipeline(rows, slots, honest, rule, H, attack, 2.0, mixing=mixing, n_perms=3,
                                                **WORDS)
            V = np.stack([rows[slots[k]] for k in honest])
            G = 2.0 * AAO.AA.gamma_of(V, "minmax_" + attack.split("_")[1])[2]
            gg = float(gams[0][j])
            i_gpu = 0 if G == 0 else int(round(gg / G * AAO.STEPS))
            top = Ob.max()
            if not np.isfinite(top):
                assert i_gpu == 0, tag
                continue
            i_or = int(np.argmax(Ob))
            if i_gpu != i_or and any(_near_tie(rows, slots, honest, attack, G * i / AAO.STEPS, H, mixing)
                                     for i in (i_gpu, i_or)):
                stats["tie"] += 1
            elif PA.margin(Ob) > MARGIN:
                assert i_gpu == i_or, f"{tag}: picked {i_gpu}, oracle {i_or}"
                stats["exact"] += 1
                stats["clipped"] += bool(((c > 0) & (c < 1)).any()) and i_gpu == int(np.argmax(Ob))
            else:
                assert Ob[i_gpu] >= top - MARGIN * abs(top), tag
                stats["near"] += 1
            stats["interior"] += 0 < i_gpu < AAO.STEPS
            stats["differs"] += gams[0][j] != gams[1][j]
    print(stats)
    assert stats["exact"] > len(cases) // 2
    assert stats["interior"] > 0 and stats["clipped"] > 0 and stats["differs"] > 0


# ---------------------------------------------------------------------------- 4. determinism and refusals
def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(11700)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _pipe_cases(rs, stack.shape[0], mixings=(None, "nnm", ("bucket", 2)))[::3][:32]
    hcases = [c[:1] + (1,) + c[2:] for c in HG._cases(rs, True) if len(c[2]) >= 5][:32]
    B = HG.Buffers(K, rs, 32)
    dst = torch.full((32, stack.shape[1]), NAN, device=K.dev)
    gam = torch.full((32, 1), NAN, device=K.dev)
    model = torch.full_like(dst, NAN)

    def run(groups):
        for x in (dst, gam, model, B.dst, B.gam, B.model):
            x.fill_(NAN)
        for g in groups:
            K.ops.pipeline_arc_attack([_pjob(K, dst[j], msgs, cases[j], gamma_out=gam[j], model_out=model[j])
                                       for j in g if j < len(cases)])
            K.ops.history_arc_attack([B.job(j, hcases[j], attack="arc_uv") for j in g if j < len(hcases)])
        return [torch.nan_to_num(x, 7.0).clone() for x in (dst, gam, model, B.dst, B.gam, B.model)]
    every = list(range(32))
    first = run([every])
    for groups in ([every], [every[::-1]], [every[5:9], every[:5], every[9:]], [[j] for j in every]):
        assert all(torch.equal(a, b) for a, b in zip(run(groups), first))


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(11800)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((4, stack.shape[1]), NAN, device=K.dev)
    gam = torch.full((4, 1), NAN, device=K.dev)
    case = ("arc_std", "clip", 1, [0, 1, -1, 3], [0, 1, 3], 300, "nnm")
    good = _pjob(K, dst[0], msgs, case, gamma_out=gam[0])
    bad = [_pjob(K, dst[1], msgs, case[:3] + ([-1, 1, 2, 3], [1, 3]) + case[5:]),   # a crafted slot 0
           _pjob(K, dst[1], msgs, case[:2] + (4,) + case[3:]),                      # H the rule refuses
           _pjob(K, dst[0], msgs, case)]                                            # overlapping dsts
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.pipeline_arc_attack([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(gam).all()
    B = HG.Buffers(K, rs, 4)
    hc = ("clip", 1, [0, 1, -1, 3], [0, 1, 3], [2], 300, 0.9, 0)
    hgood = B.job(0, hc, attack="arc_std")
    hbad = [B.job(1, ("clip", 1, [-1, 1, 2, 3], [1, 3], [0], 300, 0.9, 0), attack="arc_std"),
            B.job(1, hc, attack="arc_std", own=[1]), B.job(1, hc, attack="arc_std", dst=B.msgs[1])]
    for b in hbad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.history_arc_attack([hgood, b])
        torch.cuda.synchronize()
        assert torch.isnan(B.dst).all() and torch.isnan(B.gam).all() and torch.isnan(B.model).all()
    K.ops.pipeline_arc_attack([good])
    K.ops.history_arc_attack([hgood])
    assert torch.isfinite(dst[0, :300]).all() and torch.isfinite(B.dst[0, :300]).all()


def test_staging_bound_at_the_16_agent_team_reward_net(K):
    """n_in = 16 with 15 real slots and 1421 parameters: the history form at H = 1 (k_clip = 1, 21 rows of the 22) runs
    and its model_out is the receiver's chain."""
    rs = np.random.RandomState(11900)
    B = HG.Buffers(K, rs, 1)
    case = ("clip", 1, list(range(15)) + [-1], list(range(15)), [15], 1421, 0.9, 0)
    K.ops.history_arc_attack([B.job(0, case, attack="arc_std", dst=B.msgs[HG.N_REAL])])
    want = _hist_chain(K, B, 0, case, {15: HG.N_REAL})
    assert np.array_equal(_bits(B.model[0, :1421]), _bits(want[:1421]))


# ------------------------------------------------------------------------------------------- 5-7. Trainer
GAP = np.inf    # the oracle attacker takes the kernel's pick: ARC makes exact ties (a clipped row lies at tau from x_0,
                # as the row that set tau does), which the fp64 model of multi-Krum breaks otherwise than fp32 does;
                # the pick itself is checked against the oracle in test_pick_against_the_oracle
C2_RECEIVERS = [("clip", None, None), ("trim", None, None), ("mkrum", None, None), ("dnc", None, None),
                ("mkrum", "nnm", None), ("clip", ("bucket", 2), None), ("scclip", None, 0.9)]


@pytest.mark.parametrize("rule,mixing,momentum", C2_RECEIVERS)
def test_c2_update_round_against_the_oracle(K, rule, mixing, momentum):
    """C2 with agent 4 on arc_std (s = 2) and every cooperative agent clipping (H = 1) before `mixing` and `rule`, or
    after momentum: one update round of two epochs against the fp64 oracle through the hooks; as many launches as
    with gauss, and the kernel's gammas."""
    w, desired, _ = pretrained()
    T, N, round_ = 40, 64, 150
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=0.9, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=("arc_std", 2.0),
               aggregation=rule, momentum=momentum, clipping="arc")
    rs = np.random.RandomState(12000 + C2_RECEIVERS.index((rule, mixing, momentum)))
    rows = synth(rs, T * N)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    assert tr.arc_pairs == [0, 1, 2] and tr.arc_agents == [0, 1, 2, 3]
    agents = [AG._c2_agent(rule, w[i]) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, 0.9, dtype=f64))
    NG._follow_dnc(agents, runs)
    AG._follow_mkrum(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = AAO.chain_hook(agents, C2_BYZ, IN_NODES, {4: ("arc_std", 2.0)}, [rule] * 5, [1] * 5,
                          [momentum] * 4 + [None], [mixing] * 4 + [None], ["arc"] * 4 + [None], seed=9,
                          round_=round_, kernel_M=kernel_M, follow=follow, gammas=gammas, gap=GAP)
    want = AAO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                            common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    kg = tr.attack_gammas()
    assert sorted(kg) == sorted(gammas)
    for key, g in gammas.items():
        close(kg[key], np.asarray(g, f32), rtol=2e-3, atol=1e-6, err_msg=str(key))
    plain, _ = NG._trainer_round(dict(cfg, attack=("gauss", 1.0)), rows, round_, 2, mixing)
    assert tr.launches == plain.launches                                        # one attack launch per epoch


RULES16 = ["clip", "dnc", "trim", "wmsr", "scclip", "gmed", "mkrum", "clip"]   # the 8 cooperative agents, in order
MOM16 = [0.9, None, None, None, 0.9, None, None, None]
CLIP16 = ["arc", "arc", "arc", None, "arc", "arc", "arc", None]                # agents 3 and 7 do not clip
ARC16 = {1: ("arc_std", 2.0), 5: ("arc_uv", 2.0), 9: ("arc_sgn", 1.5), 11: ("arc_std", 1.0), 14: ("arc_uv", 0.5)}


def test_16_agent_team_with_colluding_arc_attackers(K):
    """16 agents (8 cooperative, 5 Byzantine all on arc_*, 2 Malicious, 1 Greedy; in-neighbourhoods of 8): receivers
    that clip with and without momentum hear 2-3 colluding ARC attackers each, beside receivers that do not clip.
    One update round of two epochs against the fp64 oracle: losses, weights and every pair's gamma."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, _ = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mom, clip = ["clip"] * 16, [None] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mom[i], clip[i] = RULES16[q], MOM16[q], CLIP16[q]
    H = [max(h, 1) if rules[i] == "dnc" or clip[i] else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[ARC16.get(i) for i in range(16)], momentum=mom, clipping=clip)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, None)
    assert len(tr.arc_pairs) > 8 and {clip[tr.byz_pairs[e][1]] for e in tr.arc_pairs} == {"arc", None}
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    NG._follow_dnc(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = AAO.chain_hook(agents, labels, in_nodes, ARC16, rules, H, mom, None, clip, seed=4, round_=round_,
                          kernel_M=kernel_M, follow=follow, gammas=gammas)
    want = AAO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                            common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]})")
    kg = tr.attack_gammas()
    assert sorted(kg) == sorted(gammas) and len(kg) == len(tr.arc_pairs)
    for key, g in gammas.items():
        close(kg[key], np.asarray(g, f32), rtol=2e-3, atol=1e-6, err_msg=str(key))


def test_train_rpbcac_with_an_arc_attacker(K):
    """Drop-in path: train_RPBCAC with a Byzantine_CAC_agent on ("arc_std", 2.0) against agents that clip runs the
    same rounds as a Trainer built from the same objects, bit for bit, and crafts through the ARC entry point."""
    from rcmarl import api
    from agents.adversarial_CAC_agents import Byzantine_CAC_agent
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)

    def objects():
        env, agents, args = api.build_reference_objects(cfg)
        for i in range(4):
            agents[i].clipping = "arc"
        f = agents[4]
        agents[4] = Byzantine_CAC_agent(f.actor, f.critic, f.TR, slow_lr=0.002, gamma=0.9, attack=("arc_std", 2.0))
        args["agent_label"] = C2_BYZ
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(*objects())
    tr = training.train_RPBCAC.last_trainer
    assert tr.arc_pairs == [0, 1, 2] and tr.arc_agents == [0, 1, 2, 3]
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
    assert all(np.isfinite(g).all() and (g > 0).any() for g in tr.attack_gammas().values())
