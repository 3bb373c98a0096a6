"""GPU parity of the IOS-aware Byzantine messages (rcmarl_ios_pipeline_attack, rcmarl_ios_history_attack,
include/rcmarl.h): at H = 0 bitwise the base attacks against DnC at H = 0 in all four forms; model_out bitwise the
receiver's real chain ([rcmarl_momentum_mix on a copy of M] -> [rcmarl_arc_clip] -> [rcmarl_nnm_mix] ->
rcmarl_ios_aggregate) with every crafted message sent, with and without colluders, with +-inf / 1e30 real slots, at
every H up to n_rows - 1 and at 16 slots where several removals re-centre; under bucketing sample 0 against the fp32
oracle; at scale 1 at least the min-max message's damage; the pick against the fp64 oracle
(tests/ios_attack_oracle.py) away from near ties; bitwise determinism across calls, job orders and launch splits;
refusals that leave every output untouched; and whole update rounds through Trainer -- C2 against ios receivers under
every pre-aggregation step, a 16-agent team with colluding ios_* attackers, train_RPBCAC with an ios_* Byzantine
agent, and ios_* attackers against teams without an ios receiver, which send the subset_* / arc_* messages."""
import contextlib
import io

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import arc_oracle as AO                                 # noqa: E402
import bucket_oracle as BO                              # noqa: E402
import ios_attack_oracle as IAO                         # noqa: E402
import ios_oracle as IO                                 # noqa: E402
import pipeline_attack_oracle as PA                     # noqa: E402
import subset_oracle as SO                              # noqa: E402
import team_util as TU                                  # noqa: E402
import test_arc_attack_gpu as AAG                       # noqa: E402  (the chains and the near-tie rule)
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
RULE_GAP = 1e-6                 # a removal whose ios_oracle.margin is below this may go either way in fp32
WORDS = PG.WORDS
DEVS = ("uv", "std", "sgn")


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def _cases(rs, n_rows, mixings=(None, "nnm"), colluders=False, H=None, n_ins=range(2, 17)):
    """(attack, "ios", H, slots, honest, P, mixing) at n_in 2..16: slot 0 real and honest, 1-3 crafted slots (2-3 with
    colluders), some real slots outside the honest set, H cycling 1, 2, 3, n_rows - 1 below n_rows (or the given H)."""
    out = []
    for t, n_in in enumerate(n_ins):
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
        h = max(0, min((1, 2, 3, nr - 1)[t % 4], nr - 1)) if H is None else min(H, nr - 1)
        P = int(rs.choice([33, 200, 661, 761]))
        out.append(("ios_" + DEVS[t % 3], "ios", h, slots, honest, P, mixing))
    return out


def _job(K, dst, msgs, case, scale=2.0, gamma_out=None, model_out=None, n_perms=3):
    return PG._job(K, dst, msgs, case, scale, gamma_out=gamma_out, model_out=model_out, n_perms=n_perms)


def _ios_out(K, stack, stride, P, nodes, H):
    out = torch.full((stride,), NAN, device=K.dev)
    K.ops.ios_aggregate([K.ops.vector_job(out, stack, stride, P, nodes, H, K.L.FILTER_IOS)])
    return out


def _pipe_chain(K, msgs, stride, case, sent_row, arc):
    """The receiver's chain on the stack with every crafted slot reading row sent_row: [rcmarl_arc_clip], then
    rcmarl_nnm_mix if it mixes, then rcmarl_ios_aggregate."""
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
    return _ios_out(K, stack, stride, P, nodes, H)


def _hist_chain(K, B, j, case, sent, arc):
    """The history form's receiver chain: rcmarl_momentum_mix on a copy of M, [rcmarl_arc_clip], then IOS."""
    rule, H, slots, honest, own, P, beta, first = case
    nodes = [sent[k] if s < 0 else s for k, s in enumerate(slots)]
    rows = torch.full((len(slots), HG.S), NAN, device=K.dev)
    M = B.M[j].clone()
    K.ops.momentum_mix([K.ops.momentum_job(rows, B.msgs, HG.S, P, nodes, B.ref[j], M, HG.S, beta, first)])
    if arc:
        clipped = torch.full_like(rows, NAN)
        K.ops.arc_clip([K.ops.vector_job(clipped, rows, HG.S, P, list(range(len(slots))), H, K.L.MIX_ARC)])
        rows = clipped
    return _ios_out(K, rows, HG.S, P, list(range(len(slots))), H)


def _hist_cases(rs, colluders, H=None):
    """HG._cases with the rule ios and H cycling 1, 2, 3, n_in - 1 (or the given H)."""
    out = []
    for t, c in enumerate(HG._cases(rs, colluders)):
        _, _, slots, honest, own, P, beta, first = c
        n = len(slots)
        h = min((1, 2, 3, n - 1)[t % 4], n - 1) if H is None else min(H, n - 1)
        out.append(("ios", h, slots, honest, own, P, beta, first))
    return out


# --------------------------------------------------------------------------------------------------- 1. H = 0
@pytest.mark.parametrize("arc", [0, 1])
def test_at_h0_pipeline_form_is_bitwise_the_dnc_pipeline_attack(K, arc):
    """ios x direction x mixing at n_in 2..16 with finite rows: dst, gamma_out and model_out are those of
    rcmarl_pipeline_attack (arc = 1: rcmarl_pipeline_arc_attack) against DnC at H = 0."""
    rs = np.random.RandomState(17100 + arc)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0], mixings=PG.MIXINGS, H=0, n_ins=list(range(2, 17)) * 2)
    assert {c[0] for c in cases} == set(IAO.ATTACKS)
    base = K.ops.pipeline_arc_attack if arc else K.ops.pipeline_attack
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        out = []
        for ios in (True, False):
            dst = torch.full((len(part), stack.shape[1]), NAN, device=K.dev)
            gam = torch.full((len(part), 1), NAN, device=K.dev)
            model = torch.full_like(dst, NAN)
            jobs = [_job(K, dst[j], msgs, c if ios else (("arc_" if arc else "pipeline_") + c[0].split("_")[1], "dnc")
                         + c[2:], gamma_out=gam[j], model_out=model[j]) for j, c in enumerate(part)]
            K.ops.ios_pipeline_attack(jobs, arc) if ios else base(jobs)
            out.append((dst, gam, model))
        torch.cuda.synchronize()
        for x, y in zip(*out):
            assert np.array_equal(_bits(x), _bits(y))


@pytest.mark.parametrize("arc", [0, 1])
def test_at_h0_history_form_is_bitwise_the_dnc_history_attack(K, arc):
    rs = np.random.RandomState(17200 + arc)
    cases = _hist_cases(rs, True, H=0)
    B = HG.Buffers(K, rs, 32)
    base = K.ops.history_arc_attack if arc else K.ops.history_attack
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        for d in DEVS:
            out = []
            for ios in (True, False):
                B.dst.fill_(NAN), B.gam.fill_(NAN), B.model.fill_(NAN)
                if ios:
                    K.ops.ios_history_attack([B.job(j, c, attack="ios_" + d) for j, c in enumerate(part)], arc)
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
    rs = np.random.RandomState(17300 + 4 * arc + 2 * colluders + poison)
    stack = AAG._poisoned_stack(rs, poison)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    cases = _cases(rs, n_rows, colluders=colluders, n_ins=list(range(2, 17)) * 2)
    assert {c[2] for c in cases} >= {1, 2, 3} and any(c[2] == PA.n_rows(len(c[3]), c[6]) - 1 > 3 for c in cases)
    for case in cases:
        model = torch.full((stride,), NAN, device=K.dev)
        msgs[n_rows].fill_(NAN)
        K.ops.ios_pipeline_attack([_job(K, msgs[n_rows], msgs, case, model_out=model)], arc)
        want = _pipe_chain(K, msgs, stride, case, n_rows, arc)
        torch.cuda.synchronize()
        P = case[5]
        assert np.array_equal(_bits(model[:P]), _bits(want[:P])), case
        assert torch.isnan(model[P:]).all()


@pytest.mark.parametrize("arc", [0, 1])
@pytest.mark.parametrize("colluders", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_history_form_model_out_is_what_the_receiver_computes(K, arc, colluders, poison):
    rs = np.random.RandomState(17400 + 4 * arc + 2 * colluders + poison)
    cases = [c for c in _hist_cases(rs, colluders) if len(c[2]) >= 2]
    assert {c[1] for c in cases} >= {1, 2, 3}
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
                                                 case[0], case[1], "ios_std", 2.0, B.ref[q], B.M[q], HG.S, case[6],
                                                 case[7], grp, model_out=B.model[i]))
            sent.update({k: HG.N_REAL + i for k in grp})
        K.ops.ios_history_attack(jobs, arc)
        want = _hist_chain(K, B, q, case, sent, arc)
        torch.cuda.synchronize()
        P = case[5]
        for i in range(len(groups)):
            assert np.array_equal(_bits(B.model[i, :P]), _bits(want[:P])), (case, colluders, poison)
    assert torch.equal(B.M.nan_to_num(7.0), M0.nan_to_num(7.0)) and torch.equal(B.ref, ref0)


def _recentring_stack(rs, P):
    """20 rows of P floats: honest rows near 0, two rows at +10 and one each at +2.5 and -2.0 along coordinate 0 (the
    rest small noise), so that IOS at H = 3 removes +2.5 after re-centring, where a one-shot ranking by the first
    centre would remove -2.0."""
    X = (rs.randn(20, P) * 0.05).astype(f32)
    X[12:14, 0] += 10.0
    X[14, 0] += 2.5
    X[15, 0] -= 2.0
    return X


@pytest.mark.parametrize("arc", [0, 1])
def test_16_slots_at_h3_with_removals_that_re_centre(K, arc):
    """n_in = 16 (15 real slots, one crafted) at H = 3: model_out is bitwise the chain's and, without clipping (which
    pulls the outliers in), at some pick the rows the rule reads make IOS's removals differ from a one-shot ranking by
    the first centre."""
    rs = np.random.RandomState(17500 + arc)
    P = 761
    stack = _recentring_stack(rs, P)
    msgs = torch.full((21, P), NAN, device=K.dev)
    msgs[:20] = to_dev(K, stack)[0]
    slots = list(range(11)) + [-1, 12, 13, 14, 15]
    honest = list(range(11))
    recentred = 0
    for d in DEVS:
        for scale in (0.5, 2.0):
            case = ("ios_" + d, "ios", 3, slots, honest, P, None)
            model = torch.full((P,), NAN, device=K.dev)
            gam = torch.full((1,), NAN, device=K.dev)
            K.ops.ios_pipeline_attack([_job(K, msgs[20], msgs, case, scale=scale, gamma_out=gam, model_out=model)],
                                      arc)
            want = _pipe_chain(K, msgs, P, case, 20, arc)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(model), _bits(want)), case
            Y = msgs[[20 if s < 0 else s for s in slots]].cpu().numpy().astype(f64)
            Y = AO.clip(Y, 3)[0] if arc else Y
            steps = IO.steps(Y, 3)
            d0 = steps[0][1]
            one_shot = set(sorted(d0, key=lambda k: (d0[k], k))[-3:])
            recentred += one_shot != {top for _, _, top in steps}
    assert recentred > 0 or arc


@pytest.mark.parametrize("arc", [0, 1])
def test_pipeline_form_under_bucketing_model_out_is_sample_zero(K, arc):
    """[rcmarl_arc_clip] on the slots with the crafted message, then sample 0's buckets and IOS in the fp32 oracle
    (fp64 centres and distances, the fp32 mean), where the removals' margin is clear."""
    rs = np.random.RandomState(17600 + arc)
    stack = TG._stack(rs, n_bad=0)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    cases = _cases(rs, n_rows, mixings=(("bucket", 2), ("bucket", 3)), n_ins=range(3, 17))
    checked = 0
    for case in cases:
        attack, rule, H, slots, honest, P, mixing = case
        model = torch.full((stride,), NAN, device=K.dev)
        K.ops.ios_pipeline_attack([_job(K, msgs[n_rows], msgs, case, model_out=model)], arc)
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
        if IO.margin(Z, H) < RULE_GAP:
            continue
        want = IO.aggregate(Z, H)[0]
        close(model[:P].cpu().numpy(), want, rtol=1e-5, atol=1e-6, err_msg=str(case))
        checked += 1
    assert checked > len(cases) // 2


# ------------------------------------------------------------------------------------------- 3. scale 1 vs min-max
@pytest.mark.parametrize("arc", [0, 1])
def test_at_scale_one_at_least_the_damage_of_the_minmax_message(K, arc):
    """The chain's output on dst lies at least as far from mu as its output on rcmarl_adaptive_attack's min-max
    message in the same direction (the last candidate), up to the rounding of O."""
    rs = np.random.RandomState(17700 + arc)
    stack = TG._stack(rs)
    n_rows, stride = stack.shape
    msgs = torch.full((n_rows + 1, stride), NAN, device=K.dev)
    msgs[:n_rows] = to_dev(K, stack)[0]
    mm = torch.full((stride,), NAN, device=K.dev)
    for case in _cases(rs, n_rows, n_ins=range(3, 17)):
        attack, rule, H, slots, honest, P, mixing = case
        K.ops.ios_pipeline_attack([_job(K, msgs[n_rows], msgs, case, scale=1.0)], arc)
        got = _pipe_chain(K, msgs, stride, case, n_rows, arc)[:P].cpu().numpy().astype(f64)
        K.ops.adaptive_attack([K.ops.adaptive_attack_job(mm, msgs, stride, P, [slots[k] for k in honest],
                                                         "minmax_" + attack.split("_")[1], 1.0)])
        msgs[n_rows] = mm
        ref = _pipe_chain(K, msgs, stride, case, n_rows, arc)[:P].cpu().numpy().astype(f64)
        mu = stack[[slots[k] for k in honest], :P].astype(f64).mean(0)
        o_got, o_mm = ((got - mu) ** 2).sum(), ((ref - mu) ** 2).sum()
        assert o_got >= o_mm * (1 - 1e-4) - 1e-6, case


# ------------------------------------------------------------------------------------------- 4. the pick vs fp64
def _rows_at(rows, case, g, arc, q=0):
    """The rows the rule reads at candidate gamma = g (sample q under bucketing), in fp64."""
    attack, rule, H, slots, honest, P, mixing = case
    mu, d, _ = IAO.AAO._candidates(np.stack([rows[slots[k]] for k in honest]), attack, 2.0, f64)
    m = IAO.SAO.TA.candidate(mu, d, g)
    Y = np.stack([m if s < 0 else rows[s] for s in slots])
    Y = AO.clip(Y, H)[0] if arc else Y
    bks = PA.buckets(len(slots), mixing[1], WORDS["seed"], q,
                     *[WORDS[k] for k in ("attacker", "receiver", "net", "round_", "epoch")]) \
        if isinstance(mixing, tuple) else None
    return PA.mix(Y, mixing, H, bks)


def _ios_tie(Z, H):
    """Whether IOS's removals on Z may go either way in fp32: a margin below RULE_GAP, or a step from two rows, which
    lie equally far from their mean (the fp32 rows give exactly equal d, the fp64 oracle's rows need not)."""
    return IO.margin(Z, H) < RULE_GAP or any(len(U) == 2 for U, _, _ in IO.steps(Z, H))


@pytest.mark.parametrize("arc", [0, 1])
def test_pick_against_the_oracle(K, arc):
    """The pick against the fp64 oracle with the margin rule, except where the candidates the two picks name sit at a
    near tie of IOS's removals in any shuffle sample (_ios_tie) or of the clipping or nnm order.  Among the cases there
    are interior picks and picks that differ from pipeline_*'s against DnC on the same inputs."""
    rs = np.random.RandomState(17800 + arc)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    n_rows, stride = stack.shape
    cases = _cases(rs, n_rows, mixings=(None, "nnm", ("bucket", 2)), n_ins=list(range(3, 13)) * 2)
    stats = dict(exact=0, near=0, tie=0, interior=0, differs=0)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        gams = []
        for ios in (True, False):
            dst = torch.full((len(part), stride), NAN, device=K.dev)
            gam = torch.full((len(part), 1), NAN, device=K.dev)
            if ios:
                K.ops.ios_pipeline_attack([_job(K, dst[j], msgs, c, gamma_out=gam[j]) for j, c in enumerate(part)],
                                          arc)
            else:
                base = K.ops.pipeline_arc_attack if arc else K.ops.pipeline_attack
                pre = "arc_" if arc else "pipeline_"
                base([_job(K, dst[j], msgs, (pre + c[0].split("_")[1], "dnc") + c[2:], gamma_out=gam[j])
                      for j, c in enumerate(part)])
            gams.append(gam.cpu().numpy()[:, 0])
        for j, case in enumerate(part):
            attack, rule, H, slots, honest, P, mixing = case
            tag = f"{attack} H={H} {mixing} arc={arc} slots={slots} P={P}"
            rows = stack[:, :P].astype(f64)
            _, _, Ob, _, _ = IAO.craft_pipeline(rows, slots, honest, rule, H, attack, 2.0, mixing=mixing, n_perms=3,
                                                arc=bool(arc), **WORDS)
            V = np.stack([rows[slots[k]] for k in honest])
            G = 2.0 * IAO.AAO.AA.gamma_of(V, "minmax_" + attack.split("_")[1])[2]
            gg = float(gams[0][j])
            i_gpu = 0 if G == 0 else int(round(gg / G * IAO.STEPS))
            top = Ob.max()
            if not np.isfinite(top):
                assert i_gpu == 0, tag
                continue
            i_or = int(np.argmax(Ob))

            def tied(i):
                g = G * i / IAO.STEPS
                nq = 3 if isinstance(mixing, tuple) else 1
                return (any(_ios_tie(_rows_at(rows, case, g, arc, q), H) for q in range(nq))
                        or AAG._near_tie(rows, slots, honest, attack, g, H, mixing))
            if i_gpu != i_or and (tied(i_gpu) or tied(i_or)):
                stats["tie"] += 1
            elif PA.margin(Ob) > MARGIN:
                assert i_gpu == i_or, f"{tag}: picked {i_gpu}, oracle {i_or}"
                stats["exact"] += 1
            else:
                assert Ob[i_gpu] >= top - MARGIN * abs(top), tag
                stats["near"] += 1
            stats["interior"] += 0 < i_gpu < IAO.STEPS
            stats["differs"] += gams[0][j] != gams[1][j]
    print(stats)
    assert stats["exact"] > len(cases) // 2
    assert stats["interior"] > 0 and stats["differs"] > 0


# ---------------------------------------------------------------------------- 5. determinism and refusals
def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(17900)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0], mixings=(None, "nnm", ("bucket", 2)), n_ins=list(range(3, 17)) * 3)[:32]
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
                K.ops.ios_pipeline_attack([_job(K, dst[j], msgs, cases[j], gamma_out=gam[j], model_out=model[j])
                                           for j in g if j < len(cases)], arc)
                K.ops.ios_history_attack([B.job(j, hcases[j], attack="ios_uv") for j in g if j < len(hcases)], arc)
        return [torch.nan_to_num(x, 7.0).clone() for x in (dst, gam, model, B.dst, B.gam, B.model)]
    every = list(range(32))
    first = run([every])
    for groups in ([every], [every[::-1]], [every[5:9], every[:5], every[9:]], [[j] for j in every]):
        assert all(torch.equal(a, b) for a, b in zip(run(groups), first))


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(18000)
    stack = TG._stack(rs)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((4, stack.shape[1]), NAN, device=K.dev)
    gam = torch.full((4, 1), NAN, device=K.dev)
    case = ("ios_std", "ios", 1, [0, 1, -1, 3], [0, 1, 3], 300, "nnm")
    good = _job(K, dst[0], msgs, case, gamma_out=gam[0])
    bad = [(_job(K, dst[1], msgs, case[:3] + ([-1, 1, 2, 3], [1, 3]) + case[5:]), 1),   # arc = 1, a crafted slot 0
           (_job(K, dst[1], msgs, case[:2] + (4,) + case[3:]), 0),                      # H outside [0, n_rows)
           (_job(K, dst[1], msgs, ("subset_std", "mda") + case[2:]), 0),                # not family FILTER
           (_job(K, dst[0], msgs, case), 0)]                                            # overlapping dsts
    for b, arc in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.ios_pipeline_attack([good, b], arc)
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(gam).all()
    with pytest.raises(K.L.RcmarlError):
        K.ops.ios_pipeline_attack([good], 2)
    for fn in (K.ops.pipeline_attack, K.ops.pipeline_arc_attack):                       # the base refuses FILTER
        with pytest.raises(K.L.RcmarlError):
            fn([good])
    with pytest.raises(K.L.RcmarlError):
        K.ops.subset_pipeline_attack([good], 0)
    B = HG.Buffers(K, rs, 4)
    hc = ("ios", 1, [0, 1, -1, 3], [0, 1, 3], [2], 300, 0.9, 0)
    hgood = B.job(0, hc, attack="ios_std")
    hbad = [(B.job(1, ("ios", 1, [-1, 1, 2, 3], [1, 3], [0], 300, 0.9, 0), attack="ios_std"), 1),
            (B.job(1, hc, attack="ios_std", own=[1]), 0), (B.job(1, hc, attack="ios_std", dst=B.msgs[1]), 0)]
    for b, arc in hbad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.ios_history_attack([hgood, b], arc)
        torch.cuda.synchronize()
        assert torch.isnan(B.dst).all() and torch.isnan(B.gam).all() and torch.isnan(B.model).all()
    K.ops.ios_pipeline_attack([good], 1)
    K.ops.ios_history_attack([hgood], 1)
    assert torch.isfinite(dst[0, :300]).all() and torch.isfinite(B.dst[0, :300]).all()


def test_staging_bound_at_the_16_agent_team_reward_net(K):
    """n_in = 16 with 15 real slots and 1421 parameters at H = 3: the pipeline form under nnm (37 rows, the bound) and
    the history form (22 rows, the bound) run, and their model_out is the receiver's chain."""
    rs = np.random.RandomState(18100)
    stack = TG._stack(rs, n_rows=20, P=1421)
    msgs = torch.full((21, 1421), NAN, device=K.dev)
    msgs[:20] = to_dev(K, stack)[0]
    case = ("ios_std", "ios", 3, list(range(15)) + [-1], list(range(15)), 1421, "nnm")
    model = torch.full((1421,), NAN, device=K.dev)
    K.ops.ios_pipeline_attack([_job(K, msgs[20], msgs, case, model_out=model)], 0)
    want = _pipe_chain(K, msgs, 1421, case, 20, 0)
    assert np.array_equal(_bits(model), _bits(want))
    B = HG.Buffers(K, rs, 1)
    hcase = ("ios", 3, list(range(15)) + [-1], list(range(15)), [15], 1421, 0.9, 0)
    K.ops.ios_history_attack([B.job(0, hcase, attack="ios_std", dst=B.msgs[HG.N_REAL])], 0)
    want = _hist_chain(K, B, 0, hcase, {15: HG.N_REAL}, 0)
    assert np.array_equal(_bits(B.model[0, :1421]), _bits(want[:1421]))


# ------------------------------------------------------------------------------------------- 6. Trainer
GAP = np.inf    # the oracle attacker takes the kernel's pick (checked against the oracle in test_pick_against_the_oracle)
ROUND_GAP = 1e-4
C2_RECEIVERS = [None, "nnm", "bucket", "arc", "momentum"]


def _ios_agent(w, fast, gamma, H):
    return IO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, gap=ROUND_GAP)


@pytest.mark.parametrize("pre", C2_RECEIVERS)
def test_c2_update_round_against_the_oracle(K, pre):
    """C2 with agent 4 on ios_std (s = 2) against receivers on ios at H = 1, alone, with nnm, with bucketing (s = 2),
    after clipping or momentum (0.9): one update round of two epochs against the fp64 oracle through the hooks; as
    many launches as with gauss, and the kernel's gammas."""
    w, desired, _ = pretrained()
    T, N, round_ = 40, 64, 150
    mixing = {"nnm": "nnm", "bucket": ("bucket", 2)}.get(pre)
    momentum = 0.9 if pre == "momentum" else None
    clipping = "arc" if pre == "arc" else None
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=0.9, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=("ios_std", 2.0),
               aggregation="ios", momentum=momentum, clipping=clipping)
    rs = np.random.RandomState(18200 + C2_RECEIVERS.index(pre))
    rows = synth(rs, T * N)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    assert tr.ios_pairs == [0, 1, 2] and tr.ios_agents == [0, 1, 2, 3]
    agents = [_ios_agent(w[i], 0.01, 0.9, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, 0.9, dtype=f64))
    IO.follow_kernel(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = IAO.chain_hook(agents, C2_BYZ, IN_NODES, {4: ("ios_std", 2.0)}, ["ios"] * 5, [1] * 5,
                          [momentum] * 4 + [None], [mixing] * 4 + [None], [clipping] * 4 + [None], seed=9,
                          round_=round_, kernel_M=kernel_M, follow=follow, gammas=gammas, gap=GAP)
    want = IAO.update_round(agents, C2_BYZ, IN_NODES, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
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


RULES16 = ["ios", "smea", "ios", "clip", "ios", "mda", "dnc", "ios"]           # the 8 cooperative agents, in order
MOM16 = [0.9, None, None, None, None, None, None, None]
CLIP16 = ["arc", None, "arc", "arc", None, None, None, None]
IOS16 = {1: ("ios_std", 2.0), 5: ("ios_uv", 2.0), 9: ("ios_sgn", 1.5), 11: ("ios_std", 1.0), 14: ("ios_uv", 0.5)}


def test_16_agent_team_with_colluding_ios_attackers(K):
    """16 agents (8 cooperative, 5 Byzantine all on ios_*, 2 Malicious, 1 Greedy; in-neighbourhoods of 8): receivers
    on ios with and without momentum and clipping hear 2-3 colluding ios attackers each, beside receivers on mda, smea,
    clip and dnc, which get the subset and ARC attacks' jobs.  One update round of two epochs against the fp64 oracle:
    losses, weights and every pair's gamma."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(18300)
    in_nodes, w, desired, H, fast, _ = TA._team16(rs)
    labels = TA.B16
    coop = [i for i, l in enumerate(labels) if l == "Cooperative"]
    rules, mom, clip = ["clip"] * 16, [None] * 16, [None] * 16
    for q, i in enumerate(coop):
        rules[i], mom[i], clip[i] = RULES16[q], MOM16[q], CLIP16[q]
    H = [max(h, 1) if rules[i] in ("dnc", "ios") or clip[i] else h for i, h in enumerate(H)]
    gamma, T, N, round_ = 0.9, 40, 4, 7
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               aggregation=rules, attack=[IOS16.get(i) for i in range(16)], momentum=mom, clipping=clip)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, None)
    assert len(tr.ios_pairs) > 8 and {rules[tr.byz_pairs[e][1]] for e in tr.ios_pairs} >= {"ios", "mda", "smea"}
    agents = []
    for i, lab in enumerate(labels):
        if lab == "Cooperative":
            agents.append(_ios_agent(w[i], fast[i], gamma, H[i]) if rules[i] == "ios"
                          else SO.RPBCACOracleAgent(w[i][0], w[i][1], w[i][2], 0.002, fast[i], gamma, H=H[i],
                                                    dtype=f64, aggregation=rules[i], gap=1e-4)
                          if rules[i] in SO.RULES else NG._oracle_agent(rules[i], w[i], fast[i], gamma, H[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    NG._follow_dnc(agents, runs)
    SO.follow_kernel(agents, runs)
    IO.follow_kernel(agents, runs)
    follow = {e: r.attack_gammas() for e, r in enumerate(runs)}
    gammas = {}
    hook = IAO.chain_hook(agents, labels, in_nodes, IOS16, rules, H, mom, None, clip, seed=4, round_=round_,
                          kernel_M=kernel_M, follow=follow, gammas=gammas, gap=GAP)
    want = IAO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=2, n_actor_steps=T,
                            common_reward=False, perm_source=NG._perms(), messages_hook=hook)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]}, {rules[i]})")
    kg = tr.attack_gammas()
    assert sorted(kg) == sorted(gammas) and len(kg) == len(tr.ios_pairs)
    for key, g in gammas.items():
        close(kg[key], np.asarray(g, f32), rtol=2e-3, atol=1e-6, err_msg=str(key))


@pytest.mark.parametrize("aggregation,clipping,other", [("mda", None, "subset_std"), ("smea", "arc", "subset_std"),
                                                        ("clip", "arc", "arc_std"), ("dnc", None, "arc_std")])
def test_without_an_ios_receiver_the_messages_are_the_older_attacks(K, aggregation, clipping, other):
    """C2 with agent 4 on ios_std against receivers on mda / smea (with and without clipping) or on clip / dnc: the
    round is bitwise the round with the subset_* or arc_* attacker in the same direction -- messages, gammas, weights
    and launches."""
    w, desired, _ = pretrained()
    T, N, round_ = 40, 16, 150
    rs = np.random.RandomState(18400)
    rows = synth(rs, T * N)
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=0.9, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, aggregation=aggregation,
               clipping=clipping)
    a, _ = NG._trainer_round(dict(cfg, attack=("ios_std", 2.0)), rows, round_, 2, None)
    b, _ = NG._trainer_round(dict(cfg, attack=(other, 2.0)), rows, round_, 2, None)
    torch.cuda.synchronize()
    assert a.ios_pairs == [0, 1, 2] and a.launches == b.launches
    for x, y in ((a.msg_c, b.msg_c), (a.msg_t, b.msg_t)):
        assert np.array_equal(_bits(x.nan_to_num(7.0)), _bits(y.nan_to_num(7.0)))
    ga, gb = a.attack_gammas(), b.attack_gammas()
    assert sorted(ga) == sorted(gb) and all(np.array_equal(ga[k], gb[k]) for k in ga)
    for i in range(5):
        for u, v in zip(a.get_weights(i), b.get_weights(i)):
            for x, y in zip(u, v):
                np.testing.assert_array_equal(x, y)


def test_train_rpbcac_with_an_ios_attacker(K):
    """Drop-in path: train_RPBCAC with a Byzantine_CAC_agent on ("ios_std", 2.0) against agents on ios runs the same
    rounds as a Trainer built from the same objects, bit for bit, and crafts through the IOS entry point."""
    from rcmarl import api
    from agents.adversarial_CAC_agents import Byzantine_CAC_agent
    import training.train_agents as training
    w, desired, _ = pretrained()
    cfg = dict(labels=C2_BYZ[:4] + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5, H=1,
               n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2, buffer_size=48)

    def objects():
        env, agents, args = api.build_reference_objects(cfg)
        for i in range(4):
            agents[i].aggregation = "ios"
        f = agents[4]
        agents[4] = Byzantine_CAC_agent(f.actor, f.critic, f.TR, slow_lr=0.002, gamma=0.9, attack=("ios_std", 2.0))
        args["agent_label"] = C2_BYZ
        args["n_episodes"] = 8
        args["random_seed"] = 5
        return env, agents, args
    with contextlib.redirect_stdout(io.StringIO()):
        training.train_RPBCAC(*objects())
    tr = training.train_RPBCAC.last_trainer
    assert tr.ios_pairs == [0, 1, 2] and tr.ios_agents == [0, 1, 2, 3]
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
