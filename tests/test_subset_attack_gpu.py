"""GPU parity of the subset-aware Byzantine messages (rcmarl_subset_pipeline_attack, rcmarl_subset_history_attack,
include/rcmarl.h): at H = 0 bitwise the base attacks against DnC at H = 0 in all four forms; model_out bitwise the
receiver's real chain ([rcmarl_momentum_mix on a copy of M] -> [rcmarl_arc_clip] -> [rcmarl_nnm_mix] ->
rcmarl_subset_aggregate) with every crafted message sent, with and without colluders and with +-inf / 1e30 real slots;
under bucketing sample 0 against the fp32 oracle; at scale 1 at least the min-max message's damage; the pick against
the fp64 oracle (tests/subset_attack_oracle.py) away from near ties; bitwise determinism across calls, job orders and
launch splits; refusals that leave every output untouched; and whole update rounds through Trainer -- C2 against mda
and smea receivers under every pre-aggregation step, a 16-agent team with colluding subset_* attackers, and
train_RPBCAC with a subset_* Byzantine agent."""
import contextlib
import io

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import arc_oracle as AO                                 # noqa: E402
import bucket_oracle as BO                              # noqa: E402
import pipeline_attack_oracle as PA                     # noqa: E402
import subset_attack_oracle as SAO                      # noqa: E402
import subset_oracle as SO                              # noqa: E402
import team_util as TU                                  # noqa: E402
import test_arc_attack_gpu as AAG                       # noqa: E402  (the chains and the near-tie rule)
import test_arc_gpu as AG                               # noqa: E402  (the C2 oracle agents)
import test_history_attack_gpu as HG                    # noqa: E402  (the history buffers and cases)
import test_nnm_gpu as NG                               # noqa: E402  (the C2 round helpers)
import test_pipeline_attack_gpu as PG                   # noqa: E402  (the pipeline jobs)
import test_tailored_attacks_gpu as TG                  # noqa: E402  (the message stacks)
from golden_util import pretrained                      # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                   # noqa: E402  (checker only)

f32, f64 = np.float32, np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
MARGIN = 1e-4
RULE_GAP = 1e-6                 # a selection whose subset_oracle.margin is below this may go either way in fp32
WORDS = PG.WORDS
DEVS = ("uv", "std", "sgn")


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def _cases(rs, n_rows, mixings=(None, "nnm"), colluders=False, H=None, n_ins=range(2, 17)):
    """(attack, rule, H, slots, honest, P, mixing) for mda and smea at n_in 2..16: slot 0 real and honest, 1-3 crafted
    slots (2-3 with colluders), some real slots outside the honest set, H 1..3 (or the given H) below n_rows."""
    out = []
    t = 0
    for n_in in n_ins:
        for rule in SAO.RULES:
            mixing = mixings[t % len(mixings)]
            if isinstance(mixing, tuple) and n_in < 3:
                mixing = None
            n_cr = min(1 + int(rs.randint(3)) if not colluders else 2 + int(rs.randint(2)), n_in - 1)
            real = [int(x) for x in rs.choice(n_rows, size=n_in - n_cr, replace=False)]
            if real[0] >= n_rows - 4:
                real[0] = int(rs.choice([r for r in range(n_rows - 4) if r not in real[1:]]))
            slots = real[:1] + [-1] * n_cr + real[1:]
            rest = slots[1:]
            rs.shuffle(rest)
            slots[1:] = rest
            honest = [k for k, s in enumerate(slots) if 0 <= s < n_rows - 4]
            nr = PA.n_rows(n_in, mixing)
            h = min(1 + t % 3, nr - 1) if H is None else min(H, nr - 1)
            P = int(rs.choice([33, 200, 661, 761]))
            out.append(("subset_" + DEVS[t % 3], rule, h, slots, honest, P, mixing))
            t += 1
    return out


def _job(K, dst, msgs, case, scale=2.0, gamma_out=None, model_out=None, n_perms=3):
    return PG._job(K, dst, msgs, case, scale, gamma_out=gamma_out, model_out=model_out, n_perms=n_perms)


def _subset_out(K, stack, stride, P, nodes, rule, H):
    out = torch.full((stride,), NAN, device=K.dev)
    K.ops.subset_aggregate([K.ops.vector_job(out, stack, stride, P, nodes, H, K.L.SUBSET_RULES[rule])])
    return out


def _pipe_chain(K, msgs, stride, case, sent_row, arc):
    """The receiver's chain on the stack with every crafted slot reading row sent_row: [rcmarl_arc_clip], then
    rcmarl_nnm_mix if it mixes, then rcmarl_subset_aggregate."""
    attack, rule, H, slots, honest, P, mixing = case
    stack, nodes = msgs, [sent_row if s < 0 else s for s in slots]
    if arc:
        clipped = torch.full((len(slots), stride), NAN, device=K.dev)
        K.ops.arc_clip([K.ops.vector_job(clipped, stack, stride, P, nodes, H, K.L.MIX_ARC)])
        stack, nodes = clipped, list(range(len(slots)))
    if mixing == "nnm":
        mixed = torch.full((len(slots), stride), NAN, device=K.dev)
        K.ops.nnm_mix([K.ops.vector_job(mixed, stack, stride, P, nodes, H, K.L.MIX_NNM)])
        stack, nodes = mixed, list(range(len(slots)))
    return _subset_out(K, stack, stride, P, nodes, rule, H)


def _hist_chain(K, B, j, case, sent, arc):
    """The history form's receiver chain: rcmarl_momentum_mix on a copy of M, [rcmarl_arc_clip], then the rule."""
    rule, H, slots, honest, own, P, beta, first = case
    nodes = [sent[k] if s < 0 else s for k, s in enumerate(slots)]
    rows = torch.full((len(slots), HG.S), NAN, device=K.dev)
    M = B.M[j].clone()
    K.ops.momentum_mix([K.ops.momentum_job(rows, B.msgs, HG.S, P, nodes, B.ref[j], M, HG.S, beta, first)])
    if arc:
        clipped = torch.full_like(rows, NAN)
        K.ops.arc_clip([K.ops.vector_job(clipped, rows, HG.S, P, list(range(len(slots))), H, K.L.MIX_ARC)])
        rows = clipped
    return _subset_out(K, rows, HG.S, P, list(range(len(slots))), rule, H)


def _hist_cases(rs, colluders, H=None):
    """HG._cases with the rule mda or smea (alternately) and H 1..3 below n_in (or the given H)."""
    out = []
    for t, c in enumerate(HG._cases(rs, colluders)):
        rule, _, slots, honest, own, P, beta, first = c
        h = min(1 + t % 3, len(slots) - 1) if H is None else min(H, len(slots) - 1)
        out.append((SAO.RULES[t % 2], h, slots, honest, own, P, beta, first))
    return out


# --------------------------------------------------------------------------------------------------- 1. H = 0
@pytest.mark.parametrize("arc", [0, 1])
def test_at_h0_pipeline_form_is_bitwise_the_dnc_pipeline_attack(K, arc):
    """mda and smea x direction x mixing at n_in 2..16 with finite rows: dst, gamma_out and model_out are those of
    rcmarl_pipeline_attack (arc = 1: rcmarl_pipeline_arc_attack) against DnC at H = 0."""
    rs = np.random.RandomState(15100 + arc)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0], mixings=PG.MIXINGS, H=0)
    assert {c[1] for c in cases} == set(SAO.RULES) and {c[0] for c in cases} == set(SAO.ATTACKS)
    base = K.ops.pipeline_arc_attack if arc else K.ops.pipeline_attack
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        out = []
        for sub in (True, False):
            dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
            gam = torch.full((len(part), 1), NAN, device=K.dev)
            model = torch.full_like(dst, NAN)
            jobs = [_job(K, dst[j], msgs, c if sub else (("arc_" if arc else "pipeline_") + c[0].split("_")[1], "dnc")
                         + c[2:], gamma_out=gam[j], model_out=model[j]) for j, c in enumerate(part)]
            K.ops.subset_pipeline_attack(jobs, arc) if sub else base(jobs)
            out.append((dst, gam, model))
        torch.cuda.synchronize()
        for x, y in zip(*out):
            assert np.array_equal(_bits(x), _bits(y))


@pytest.mark.parametrize("arc", [0, 1])
def test_at_h0_history_form_is_bitwise_the_dnc_history_attack(K, arc):
    rs = np.random.RandomState(15200 + arc)
    cases = _hist_cases(rs, True, H=0)
    B = HG.Buffers(K, rs, 32)
    base = K.ops.history_arc_attack if arc else K.ops.history_attack
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        for d in DEVS:
            out = []
            for sub in (True, False):
                B.dst.fill_(NAN), B.gam.fill_(NAN), B.model.fill_(NAN)
                if sub:
                    K.ops.subset_history_attack([B.job(j, c, attack="subset_" + d) for j, c in enumerate(part)], arc)
                else:
                    base([B.job(j, ("dnc",) + c[1:], attack=("arc_" if arc else "history_") + d)
                          for j, c in enumerate(part)])
                out.append([x.clone() for x in (B.dst, B.gam, B.model)])
            torch.cuda.synchronize()
            for x, y in zip(*out):
                assert np.array_equal(_bits(x), _bits(y)), d


# ----------------------------------------------------------------------------------------- 2. model_out = the chain
@pytest.mark.parametrize("arc", [0, 1])
@pytest.mark.parametrize("colluders", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_pipeline_form_model_out_is_what_the_receiver_computes(K, arc, colluders, poison):
    rs = np.random.RandomState(15300 + 4 * arc + 2 * colluders + poison)
    stack = AAG._poisoned_stack(rs, poison)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    cases = _cases(rs, n_rows, colluders=colluders, n_ins=range(3, 17))
    assert {c[1] for c in cases} == set(SAO.RULES) and {c[2] for c in cases} == {1, 2, 3}
    for case in cases:
        model = torch.full((stride,), NAN, device=K.dev)
        msgs[n_rows].fill_(NAN)
        K.ops.subset_pipeline_attack([_job(K, msgs[n_rows], msgs, case, model_out=model)], arc)
        want = _pipe_chain(K, msgs, stride, case, n_rows, arc)
        torch.cuda.synchronize()
        P = case[5]
        assert np.array_equal(_bits(model[:P]), _bits(want[:P])), case
        assert torch.isnan(model[P:]).all()


@pytest.mark.parametrize("arc", [0, 1])
@pytest.mark.parametrize("colluders", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_history_form_model_out_is_what_the_receiver_computes(K, arc, colluders, poison):
    rs = np.random.RandomState(15400 + 4 * arc + 2 * colluders + poison)
    cases = [c for c in _hist_cases(rs, colluders) if len(c[2]) >= 3]
    assert {c[0] for c in cases} == set(SAO.RULES) and {c[1] for c in cases} == {1, 2, 3}
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
                                                 case[0], case[1], "subset_std", 2.0, B.ref[q], B.M[q], HG.S, case[6],
                                                 case[7], grp, model_out=B.model[i]))
            sent.update({k: HG.N_REAL + i for k in grp})
        K.ops.subset_history_attack(jobs, arc)
        want = _hist_chain(K, B, q, case, sent, arc)
        torch.cuda.synchronize()
        P = case[5]
        for i in range(len(groups)):
            assert np.array_equal(_bits(B.model[i, :P]), _bits(want[:P])), (case, colluders, poison)
    assert torch.equal(B.M.nan_to_num(7.0), M0.nan_to_num(7.0)) and torch.equal(B.ref, ref0)


@pytest.mark.parametrize("arc", [0, 1])
def test_pipeline_form_under_bucketing_model_out_is_sample_zero(K, arc):
    """[rcmarl_arc_clip] on the slots with the crafted message, then sample 0's buckets and MDA / SMEA in the fp32
    oracle (fp64 distances, the fp32 mean), where the selection's margin is clear."""
    rs = np.random.RandomState(15500 + arc)
    stack = TG._stack(rs, n_bad=0)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    cases = _cases(rs, n_rows, mixings=(("bucket", 2), ("bucket", 3)), n_ins=range(3, 17))
    checked = 0
    for case in cases:
        attack, rule, H, slots, honest, P, mixing = case
        model = torch.full((stride,), NAN, device=K.dev)
        K.ops.subset_pipeline_attack([_job(K, msgs[n_rows], msgs, case, model_out=model)], arc)
        nodes = [n_rows if s < 0 else s for s in slots]
        if arc:
            clipped = torch.full((len(slots), stride), NAN, device=K.dev)
            K.ops.arc_clip([K.ops.vector_job(clipped, msgs, stride, P, nodes, H, K.L.MIX_ARC)])
            Y = clipped[:, :P].cpu().numpy()
        else:
            Y = msgs[nodes, :P].cpu().numpy()
        bks = PA.buckets(len(slots), mixing[1], WORDS["seed"], 0,
                         *[WORDS[k] for k in ("attacker", "receiver", "net", "round_", "epoch")])
        Z = BO.mix(Y, bks)[0]
        if SO.margin(rule, Z, H) < RULE_GAP:
            continue
        want = SO.aggregate(rule, Z, H)[0]
        close(model[:P].cpu().numpy(), want, rtol=1e-5, atol=1e-6, err_msg=str(case))
        checked += 1
    assert checked > len(cases) // 2


# ------------------------------------------------------------------------------------------- 3. scale 1 vs min-max
@pytest.mark.parametrize("arc", [0, 1])
def test_at_scale_one_at_least_the_damage_of_the_minmax_message(K, arc):
    """The chain's output on dst lies at least as far from mu as its output on rcmarl_adaptive_attack's min-max
    message in the same direction (the last candidate), up to the rounding of O."""
    rs = np.random.RandomState(15600 + arc)
    stack = TG._stack(rs)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    mm = torch.full((stride,), NAN, device=K.dev)
    for case in _cases(rs, n_rows, n_ins=range(3, 17)):
        attack, rule, H, slots, honest, P, mixing = case
        K.ops.subset_pipeline_attack([_job(K, msgs[n_rows], msgs, case, scale=1.0)], arc)
        got = _pipe_chain(K, msgs, stride, case, n_rows, arc)[:P].cpu().numpy().astype(f64)
        K.ops.adaptive_attack([K.ops.adaptive_attack_job(mm, msgs, stride, P, [slots[k] for k in honest],
                                                         "minmax_" + attack.split("_")[1], 1.0)])
        msgs[n_rows] = mm
        ref = _pipe_chain(K, msgs, stride, case, n_rows, arc)[:P].cpu().numpy().astype(f64)
        mu = stack[[slots[k] for k in honest], :P].astype(f64).mean(0)
        o_got, o_mm = ((got - mu) ** 2).sum(), ((ref - mu) ** 2).sum()
        assert o_got >= o_mm * (1 - 1e-4) - 1e-6, case


# ------------------------------------------------------------------------------------------- 4. the pick vs fp64
def _rows_at(rows, case, g, arc):
    """The rows the rule reads at candidate gamma = g (sample 0 under bucketing), in fp64."""
    attack, rule, H, slots, honest, P, mixing = case
    mu, d, _ = SAO.AAO._candidates(np.stack([rows[slots[k]] for k in honest]), attack, 2.0, f64)
    m = SAO.TA.candidate(mu, d, g)
    Y = np.stack([m if s < 0 else rows[s] for s in slots])
    Y = AO.clip(Y, H)[0] if arc else Y
    bks = PA.buckets(len(slots), mixing[1], WORDS["seed"], 0,
                     *[WORDS[k] for k in ("attacker", "receiver", "net", "round_", "epoch")]) \
        if isinstance(mixing, tuple) else None
    return PA.mix(Y, mixing, H, bks)


@pytest.mark.parametrize("arc", [0, 1])
def test_pick_against_the_oracle(K, arc):
    """The pick against the fp64 oracle with the margin rule, except where the candidates the two picks name sit at a
    near tie of the subset selection (subset_oracle.margin below RULE_GAP) or of the clipping or nnm order.  Among the
    cases there are interior picks and picks that differ from pipeline_*'s against DnC on the same inputs."""
    rs = np.random.RandomState(15700 + arc)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    n_rows, stride = stack.shape
    cases = _cases(rs, n_rows, mixings=(None, "nnm", ("bucket", 2)), n_ins=range(3, 13))
    stats = dict(exact=0, near=0, tie=0, interior=0, differs=0)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        gams = []
        for sub in (True, False):
            dst = torch.full((len(part), stride), NAN, device=K.dev)
            gam = torch.full((len(part), 1), NAN, device=K.dev)
            if sub:
                K.ops.subset_pipeline_attack([_job(K, dst[j], msgs, c, gamma_out=gam[j]) for j, c in enumerate(part)],
                                             arc)
            else:
                base = K.ops.pipeline_arc_attack if arc else K.ops.pipeline_attack
                pre = "arc_" if arc else "pipeline_"
                base([_job(K, dst[j], msgs, (pre + c[0].split("_")[1], "dnc") + c[2:], gamma_out=gam[j])
                      for j, c in enumerate(part)])
            gams.append(gam.cpu().numpy()[:, 0])
        for j, case in enumerate(part):
            attack, rule, H, slots, honest, P, mixing = case
            tag = f"{attack} {rule} H={H} {mixing} arc={arc} slots={slots} P={P}"
            rows = stack[:, :P].astype(f64)
            _, _, Ob, _, _ = SAO.craft_pipeline(rows, slots, honest, rule, H, attack, 2.0, mixing=mixing, n_perms=3,
                                                arc=bool(arc), **WORDS)
            V = np.stack([rows[slots[k]] for k in honest])
            G = 2.0 * SAO.AAO.AA.gamma_of(V, "minmax_" + attack.split("_")[1])[2]
            gg = float(gams[0][j])
            i_gpu = 0 if G == 0 else int(round(gg / G * SAO.STEPS))
            top = Ob.max()
            if not np.isfinite(top):
                assert i_gpu == 0, tag
                continue
            i_or = int(np.argmax(Ob))

            def tied(i):
                g = G * i / SAO.STEPS
                return (SO.margin(rule, _rows_at(rows, case, g, arc), H) < RULE_GAP
                        or AAG._near_tie(rows, slots, honest, attack, g, H, mixing))
            if i_gpu != i_or and (tied(i_gpu) or tied(i_or)):
                stats["tie"] += 1
            elif PA.margin(Ob) > MARGIN:
                assert i_gpu == i_or, f"{tag}: picked {i_gpu}, oracle {i_or}"
                stats["exact"] += 1
            else:
                assert Ob[i_gpu] >= top - MARGIN * abs(top), tag
                stats["near"] += 1
            stats["interior"] += 0 < i_gpu < SAO.STEPS
            stats["differs"] += gams[0][j] != gams[1][j]
    print(stats)
    assert stats["exact"] > len(cases) // 2
    assert stats["interior"] > 0 and stats["differs"] > 0


# ---------------------------------------------------------------------------- 5. determinism and refusals
def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(15800)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0], mixings=(None, "nnm", ("bucket", 2)), n_ins=list(range(3, 17)) * 2)[:32]
    hcases = [c for c in _hist_cases(rs, True) if len(c[2]) >= 3][:32]
    B = HG.Buffers(K, rs, 32)
    dst = torch.full((32, stack.shape[1]), NAN, device=K.dev)
    gam = torch.full((32, 1), NAN, device=K.dev)
    model = torch.full_like(dst, NAN)

    def run(groups):
        for x in (dst, gam, model, B.dst, B.gam, B.model):
            x.fill_(NAN)
        for g in groups:
            for arc in (0, 1):                          # arc = 1 overwrites arc = 0: both must be deterministic
                K.ops.subset_pipeline_attack([_job(K, dst[j], msgs, cases[j], gamma_out=gam[j], model_out=model[j])
                                              for j in g if j < len(cases)], arc)
                K.ops.subset_history_attack([B.job(j, hcases[j], attack="subset_uv") for j in g if j < len(hcases)],
                                            arc)
        return [torch.nan_to_num(x, 7.0).clone() for x in (dst, gam, model, B.dst, B.gam, B.model)]
    every = list(range(32))
    first = run([every])
    for groups in ([every], [every[::-1]], [every[5:9], every[:5], every[9:]], [[j] for j in every]):
        assert all(torch.equal(a, b) for a, b in zip(run(groups), first))


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(15900)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((4, stack.shape[1]), NAN, device=K.dev)
    gam = torch.full((4, 1), NAN, device=K.dev)
    case = ("subset_std", "mda", 1, [0, 1, -1, 3], [0, 1, 3], 300, "nnm")
    good = _job(K, dst[0], msgs, case, gamma_out=gam[0])
    bad = [(_job(K, dst[1], msgs, case[:3] + ([-1, 1, 2, 3], [1, 3]) + case[5:]), 1),   # arc = 1, a crafted slot 0
           (_job(K, dst[1], msgs, case[:2] + (4,) + case[3:]), 0),                      # H outside [0, n_rows)
           (_job(K, dst[1], msgs, ("pipeline_std", "clip") + case[2:]), 0),             # not family SUBSET
           (_job(K, dst[0], msgs, case), 0)]                                            # overlapping dsts
    for b, arc in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.subset_pipeline_attack([good, b], arc)
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(gam).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.subset_pipeline_attack([good], 2)
    with pytest.raises(K.L.RcmarlError):
        K.ops.pipeline_attack([good])                                                   # the base refuses SUBSET
    B = HG.Buffers(K, rs, 4)
    hc = ("smea", 1, [0, 1, -1, 3], [0, 1, 3], [2], 300, 0.9, 0)
    hgood = B.job(0, hc, attack="subset_std")
    hbad = [(B.job(1, ("smea", 1, [-1, 1, 2, 3], [1, 3], [0], 300, 0.9, 0), attack="subset_std"), 1),
            (B.job(1, hc, attack="subset_std", own=[1]), 0), (B.job(1, hc, attack="subset_std", dst=B.msgs[1]), 0)]
    for b, arc in hbad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.subset_history_attack([hgood, b], arc)
        torch.cuda.synchronize()
        assert torch.isnan(B.dst).all() and torch.isnan(B.gam).all() and torch.isnan(B.model).all()
    K.ops.subset_pipeline_attack([good], 1)
    K.ops.subset_history_attack([hgood], 1)
    assert torch.isfinite(dst[0, :300]).all() and torch.isfinite(B.dst[0, :300]).all()


@pytest.mark.parametrize("rule", SAO.RULES)
def test_staging_bound_at_the_16_agent_team_reward_net(K, rule):
    """n_in = 16 with 15 real slots and 1421 parameters at H = 1: the pipeline form under nnm (35 rows, the bound) and
    the history form with ARC (k_clip = 1, 21 rows) run, and their model_out is the receiver's chain."""
    rs = np.random.RandomState(16000 + len(rule))
    stack = TG._stack(rs, n_rows=20, P=1421)
    msgs = torch.full((21, 1421), NAN, device=K.dev)
    msgs[:20] = to_dev(K, stack)[0]
    case = ("subset_std", rule, 1, list(range(15)) + [-1], list(range(15)), 1421, "nnm")
    model = torch.full((1421,), NAN, device=K.dev)
    K.ops.subset_pipeline_attack([_job(K, msgs[20], msgs, case, model_out=model)], 0)
    want = _pipe_chain(K, msgs, 1421, case, 20, 0)
    assert np.array_equal(_bits(model), _bits(want))
    B = HG.Buffers(K, rs, 1)
    hcase = (rule, 1, list(range(15)) + [-1], list(range(15)), [15], 1421, 0.9, 0)
    K.ops.subset_history_attack([B.job(0, hcase, attack="subset_std", dst=B.msgs[HG.N_REAL])], 1)
    want = _hist_chain(K, B, 0, hcase, {15: HG.N_REAL}, 1)
    assert np.array_equal(_bits(B.model[0, :1421]), _bits(want[:1421]))


# ------------------------------------------------------------------------------------------- 6. Trainer
GAP = np.inf    # the oracle attacker takes the kernel's pick (checked against the oracle in test_pick_against_the_oracle)
C2_RECEIVERS = [(rule, pre) for rule in SAO.RULES for pre in (None, "nnm", "bucket", "momentum", "arc")]


def _c2_agent(rule, w):
    if rule == "mda":
        return AG.MdaAgent(w[0], w[1], w[2], 0.002, 0.01, 0.9, H=1, dtype=f64, aggregation=rule, gap=1e-4)
    return SO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, 0.01, 0.9, H=1, dtype=f64, aggregation=rule, gap=1e-4)


@pytest.mark.parametrize("rule,pre", C2_RECEIVERS)
def test_c2_update_round_against_the_oracle(K, rule, pre):
    """C2 with agent 4 on subset_std (s = 2) against receivers on `rule` at H = 1, alone, with nnm, with bucketing
    (s = 2), after momentum (0.9) or clipping: one update round of two epochs against the fp64 oracle through the hooks;
    as many launches as with gauss, and the kernel's gammas."""
    w, desired, _ = pretrained()
    T, N, round_ = 40, 64, 150
    mixing = {"nnm": "nnm", "bucket": ("bucket", 2)}.get(pre)
    momentum = 0.9 if pre == "momentum" else None
    clipping = "arc" if pre == "arc" else None
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=0.9, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=("subset_std", 2.0),
               aggregation=rule, momentum=momentum, clipping=clipping)
    rs = np.random.RandomState(16100 + C2_RECEIVERS.index((rule, pre)))
    rows = synth(rs, T * N)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    assert tr.subset_pairs == [0, 1, 2] and tr.subset_agents == [0, 1, 2, 3]
    agents = [_c2_agent(rule, w[i]) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, 0.9, dtype=f64))
    SO.follow_kernel(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = SAO.chain_hook(agents, C2_BYZ, IN_NODES, {4: ("subset_std", 2.0)}, [rule] * 5, [1] * 5,
                          [momentum] * 4 + [None], [mixing] * 4 + [None], [clipping] * 4 + [None], seed=9,
                          round_=round_, kernel_M=kernel_M, follow=follow, gammas=gammas, gap=GAP)
    want = SAO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
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


RULES16 = ["mda", "smea", "mda", "clip", "smea", "mda", "dnc", "smea"]         # the 8 cooperative agents, in order
MOM16 = [0.9, None, None, None, 0.9, None, None, None]
CLIP16 = ["arc", None, "arc", "arc", None, None, None, "arc"]
SUB16 = {1: ("subset_std", 2.0), 5: ("subset_uv", 2.0), 9: ("subset_sgn", 1.5), 11: ("subset_std", 1.0),
         14: ("subset_uv", 0.5)}


def test_16_agent_team_with_colluding_subset_attackers(K):
    """16 agents (8 cooperative, 5 Byzantine all on subset_*, 2 Malicious, 1 Greedy; in-neighbourhoods of 8):
    receivers on mda and smea with and without momentum and clipping hear 2-3 colluding subset attackers each, beside
    receivers on clip and dnc, which get the ARC attack's jobs.  One update round of two epochs against the fp64 oracle:
    losses, weights and every pair's gamma."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(16200)
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
               aggregation=rules, attack=[SUB16.get(i) for i in range(16)], momentum=mom, clipping=clip)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, None)
    assert len(tr.subset_pairs) > 8 and {rules[tr.byz_pairs[e][1]] for e in tr.subset_pairs} >= {"mda", "smea"}
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(SO.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, fast[i], gamma, H=H[i], dtype=f64,
                                               aggregation=rules[i], gap=1e-4) if rules[i] in SAO.RULES
                          else NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    NG._follow_dnc(agents, runs)
    SO.follow_kernel(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = SAO.chain_hook(agents, labels, in_nodes, SUB16, rules, H, mom, None, clip, seed=4, round_=round_,
                          kernel_M=kernel_M, follow=follow, gammas=gammas, gap=GAP)
    want = SAO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                            common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]})")
    kg = tr.attack_gammas()
    assert sorted(kg) == sorted(gammas) and len(kg) == len(tr.subset_pairs)
    for key, g in gammas.items():
        close(kg[key], np.asarray(g, f32), rtol=2e-3, atol=1e-6, err_msg=str(key))


def test_train_rpbcac_with_a_subset_attacker(K):
    """Drop-in path: train_RPBCAC with a Byzantine_CAC_agent on ("subset_std", 2.0) against agents on mda runs the same
    rounds as a Trainer built from the same objects, bit for bit, and crafts through the subset entry point."""
    from rcmarl import api
    from agents.adversarial_CAC_agents import Byzantine_CAC_agent
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)

    def objects():
        env, agents, args = api.build_reference_objects(cfg)
        for i in range(4):
            agents[i].aggregation = "mda"
        f = agents[4]
        agents[4] = Byzantine_CAC_agent(f.actor, f.critic, f.TR, slow_lr=0.002, gamma=0.9, attack=("subset_std", 2.0))
        args["agent_label"] = C2_BYZ
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(*objects())
    tr = training.train_RPBCAC.last_trainer
    assert tr.subset_pairs == [0, 1, 2] and tr.subset_agents == [0, 1, 2, 3]
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
