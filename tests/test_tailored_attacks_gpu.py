"""GPU parity of the rule-aware Byzantine messages (rcmarl_tailored_attack, include/rcmarl.h) against the fp64 oracle
(tests/tailored_attack_oracle.py): the kernel for every rule x every direction, n_in 2..16 with 1-3 crafted slots and
Malicious-style real slots, the trainer's parameter counts, 32 jobs per launch with gamma_out; scale 0 against
rcmarl_attack's ALIE at z = 0 and a plain-mean receiver against rcmarl_adaptive_attack's min-max, bit for bit; bitwise
determinism; a job at the staging bound as the first launch of a fresh process; the refusals; whole update rounds
through Trainer (the C2 team with agent 4 on each tailored attack under each rule, a 16-agent team with colluding
tailored attackers, a world-1 PeerComm) and Trainer.attack_gammas.

Margins.  The kernel picks i* = argmax_i O_i of fp32 objectives; the oracle's are fp64.  Where the oracle's relative
margin between its best and its second-best distinct objective exceeds MARGIN = 1e-4, the kernel's pick must be the
oracle's, exactly (an exact tie, e.g. a plateau where the crafted slot is trimmed or not selected for every larger gamma,
is shared by fp32 and must go to the smaller i).  Otherwise the fp64 objective of the kernel's pick must be within
MARGIN relative of the maximum.  gamma_mm itself carries fp32 rounding (rtol G_RTOL = 5e-5, as the min-max tests), so
the kernel's gamma is matched to the oracle's candidate of the same index, and the message is compared at the fp32
tolerances of test_adaptive_attacks_gpu.py.  After whole update rounds the honest messages carry the round's fp32 error:
weights rtol 1e-3 / atol 5e-5, losses rtol 2e-3 / atol 2e-5, and gamma rtol 2e-3 where the oracle's margin exceeds
MARGIN (the per-case minimum margin is printed)."""
import datetime
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                     # noqa: E402
import agg_oracle as AO                                 # noqa: E402
import attack_oracle as AT                              # noqa: E402
import tailored_attack_oracle as TA                     # noqa: E402
import team_util as TU                                  # noqa: E402
import vector_oracle as VO                              # noqa: E402
from golden_util import pretrained                      # noqa: E402
from kernel_util import close, load_kernels, to_dev     # noqa: E402
from oracle import rpbcac_oracle as O                   # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
C2_BYZ = ["Cooperative"] * 4 + ["Byzantine"]
PAR_COUNTS = (661, 761, 1101, 1421)
MARGIN = 1e-4
G_RTOL = 5e-5
_T0 = time.time()


@pytest.fixture(scope="module")
def K():
    yield load_kernels()
    print(f"\ntest_tailored_attacks_gpu.py: {time.time() - _T0:.1f} s")


def msg_atol(vmax, g, dmax):
    return 1e-5 * max(vmax, 1.0) + G_RTOL * g * dmax


def _max_h(rule, n_in):
    if rule in ("krum", "mkrum"):
        return n_in - 3
    if rule == "trim":
        return (n_in - 1) // 2
    return n_in - 1


# ---------------------------------------------------------------------------------------------------------- kernel
def _stack(rs, n_rows=24, P=max(PAR_COUNTS), n_bad=4):
    """Messages around a common centre, each row with its own spread; the last n_bad rows are Malicious-style (far
    from the centre)."""
    centre = rs.randn(P)
    X = centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))
    X[n_rows - n_bad:] += rs.randn(n_bad, P) * 3.0
    return X.astype(np.float32)


def _cases(rs, n_rows, n_bad=4):
    """(attack, rule, H, slots, honest, P) for every rule x direction at n_in 2..16, 1-3 crafted slots, some real slots
    Malicious-style"""
    out = []
    c = 0
    for rule in TA.RULES:
        for attack in TA.ATTACKS:
            for n_in in (2, 3, 4, 5, 7, 10, 13, 16):
                if rule in ("krum", "mkrum") and n_in < 3:
                    continue
                n_cr = min(1 + c % 3, n_in - 1)
                n_mal = min(c % 2 + (n_in > 6), n_in - 1 - n_cr)
                n_hon = n_in - n_cr - n_mal
                hon_rows = [int(x) for x in rs.choice(n_rows - n_bad, size=n_hon, replace=False)]
                mal_rows = [int(x) for x in rs.choice(range(n_rows - n_bad, n_rows), size=n_mal)]
                kinds = ["c"] * n_cr + ["m"] * n_mal + ["h"] * (n_hon - 1)
                rs.shuffle(kinds)
                kinds = ["h"] + kinds                       # slot 0 is the receiver: honest
                slots, honest, ih, im = [], [], 0, 0
                for k, t in enumerate(kinds):
                    if t == "c":
                        slots.append(-1)
                    elif t == "m":
                        slots.append(mal_rows[im]); im += 1
                    else:
                        slots.append(hon_rows[ih]); ih += 1
                        honest.append(k)
                H = int(rs.randint(0, _max_h(rule, n_in) + 1))
                out.append((attack, rule, H, slots, honest, PAR_COUNTS[c % 4]))
                c += 1
    return out


def _launch(K, msgs, stride, cases, scale=2.0):
    dst = torch.full((len(cases), stride), NAN, device=K.dev)
    gam = torch.full((len(cases), 2), NAN, device=K.dev)
    jobs = [K.ops.tailored_attack_job(dst[j], msgs, stride, P, slots, honest, rule, H, attack, scale,
                                      gamma_out=gam[j, :1])
            for j, (attack, rule, H, slots, honest, P) in enumerate(cases)]
    return dst, gam, jobs


def _check_job(got, gg, stack, case, scale, stats):
    attack, rule, H, slots, honest, P = case
    rows = stack[:, :P].astype(f64)
    want, g, Ov = TA.craft(rows, slots, honest, rule, H, attack, scale)
    V = np.stack([rows[slots[k]] for k in honest])
    mu, d, g_mm = AA.gamma_of(V, "minmax_" + attack.split("_")[1])
    G = scale * g_mm
    tag = f"{attack} {rule} H={H} slots={slots} honest={honest} P={P}"
    assert np.isnan(got[P:]).all() and np.isnan(gg[1]), f"{tag}: wrote past n / gamma_out"
    if G == 0:
        assert gg[0] == 0, tag
        i_gpu = 0
    else:
        i_gpu = int(round(float(gg[0]) / G * TA.STEPS))
        close(gg[0], G * i_gpu / TA.STEPS, rtol=G_RTOL, atol=0, err_msg=tag)
    i_or = int(np.argmax(Ov))
    m = TA.margin(Ov)
    if m > MARGIN:
        assert i_gpu == i_or, f"{tag}: picked {i_gpu}, oracle {i_or} (margin {m:.3g}); O = {Ov}"
        stats["exact"] += 1
    else:
        top = Ov.max()
        assert Ov[i_gpu] >= top - MARGIN * abs(top), f"{tag}: O[{i_gpu}] = {Ov[i_gpu]} vs max {top}"
        stats["near"] += 1
    gi = G * i_gpu / TA.STEPS
    atol = msg_atol(np.abs(V).max(), gi, np.abs(d).max())
    close(got[:P], TA.candidate(mu, d, gi), rtol=0, atol=atol, err_msg=tag)
    stats["interior"] += 0 < i_gpu < TA.STEPS
    stats["top"] += i_gpu == TA.STEPS


@pytest.mark.parametrize("scale", [1.0, 2.0])
def test_tailored_attack_against_the_oracle(K, scale):
    """Every rule x direction at n_in 2..16 with 1-3 crafted and some Malicious-style real slots, the trainer's
    parameter counts; launches of exactly 32 jobs; the pick, gamma_out and the message against the fp64 oracle."""
    rs = np.random.RandomState(5100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])
    assert len(cases) == 162
    cases = cases + cases[:-len(cases) % 32]           # every generated case, the last launch padded to 32 jobs
    stats = dict(exact=0, near=0, interior=0, top=0)
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        dst, gam, jobs = _launch(K, msgs, stack.shape[1], part, scale)
        K.ops.tailored_attack(jobs)
        got, gg = dst.cpu().numpy(), gam.cpu().numpy()
        for j, case in enumerate(part):
            _check_job(got[j], gg[j], stack, case, scale, stats)
    print(f"{len(cases)} jobs: {stats}")
    assert stats["exact"] > len(cases) // 2 and stats["interior"] > 0 and stats["top"] > 0


def test_scale_zero_is_alie_at_z_zero_bitwise(K):
    rs = np.random.RandomState(5150)
    stack = _stack(rs)
    stack[3, :50] = 0.0
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])[::5][:32]
    dst, gam, jobs = _launch(K, msgs, stack.shape[1], cases, scale=0.0)
    K.ops.tailored_attack(jobs)
    ref = torch.full_like(dst, NAN)
    K.ops.attack([K.ops.attack_job(ref[j], msgs, stack.shape[1], P, [slots[k] for k in honest], "alie", 0.0)
                  for j, (_, _, _, slots, honest, P) in enumerate(cases)])
    torch.cuda.synchronize()
    a, b = torch.nan_to_num(dst, 7.0).cpu().numpy(), torch.nan_to_num(ref, 7.0).cpu().numpy()
    assert a.view(np.uint32).tolist() == b.view(np.uint32).tolist()
    assert (gam[:, 0] == 0).all()


@pytest.mark.parametrize("scale", [1.0, 2.0, 0.75])
def test_plain_mean_receiver_is_the_minmax_message_bitwise(K, scale):
    """A clip H = 0 receiver whose real slots are all honest: O rises strictly with i (the fp32 oracle confirms it on
    this data), so the message is rcmarl_adaptive_attack's min-max message at the same scale, bit for bit."""
    rs = np.random.RandomState(5200 + int(scale * 4))
    stack = _stack(rs, n_bad=0)
    msgs = to_dev(K, stack)[0]
    cases = []
    for j in range(32):
        n_in = 3 + j % 14                                  # at least two honest slots: gamma_mm > 0
        n_cr = 1 + j % min(3, n_in - 2)
        rows = [int(x) for x in rs.choice(stack.shape[0], size=n_in - n_cr, replace=False)]
        slots = rows[:1] + [-1] * n_cr + rows[1:]
        honest = [k for k, s in enumerate(slots) if s >= 0]
        cases.append((TA.ATTACKS[j % 3], "clip", 0, slots, honest, PAR_COUNTS[j % 4]))
    for attack, rule, H, slots, honest, P in cases:
        O32 = TA.craft(stack[:, :P], slots, honest, rule, H, attack, scale)[2]
        assert (np.diff(O32) > 0).all(), (attack, slots, O32)
    dst, gam, jobs = _launch(K, msgs, stack.shape[1], cases, scale)
    K.ops.tailored_attack(jobs)
    ref = torch.full_like(dst, NAN)
    rg = torch.full_like(gam, NAN)
    K.ops.adaptive_attack([K.ops.adaptive_attack_job(ref[j], msgs, stack.shape[1], P, [slots[k] for k in honest],
                                                      "minmax_" + attack.split("_")[1], scale, gamma_out=rg[j, :1])
                           for j, (attack, _, _, slots, honest, P) in enumerate(cases)])
    torch.cuda.synchronize()
    a, b = torch.nan_to_num(dst, 7.0).cpu().numpy(), torch.nan_to_num(ref, 7.0).cpu().numpy()
    g, r = gam[:, 0].cpu().numpy(), (torch.tensor(scale, device=K.dev) * rg[:, 0]).cpu().numpy()
    assert np.array_equal(g, r), (g, r)
    for j in range(len(cases)):
        assert a[j].view(np.uint32).tolist() == b[j].view(np.uint32).tolist(), (j, cases[j])


def test_a_range_that_overflows_fp32_sends_mu(K):
    """s * gamma_mm beyond the fp32 range: Gamma = 0, so every candidate is mu and gamma_out is 0 (not NaN)."""
    rs = np.random.RandomState(5250)
    stack = _stack(rs, n_bad=0) * 8.0                    # gamma_mm well above 1
    msgs = to_dev(K, stack)[0]
    cases = [(a, r, 0, [0, -1, 1, 2, 3], [0, 2, 3, 4], 761) for a in TA.ATTACKS for r in ("clip", "gmed")]
    dst, gam, jobs = _launch(K, msgs, stack.shape[1], cases, scale=3e38)
    K.ops.tailored_attack(jobs)
    ref = torch.full_like(dst, NAN)
    K.ops.attack([K.ops.attack_job(ref[j], msgs, stack.shape[1], P, [slots[k] for k in honest], "alie", 0.0)
                  for j, (_, _, _, slots, honest, P) in enumerate(cases)])
    torch.cuda.synchronize()
    for j, (attack, rule, H, slots, honest, P) in enumerate(cases):
        V = stack[[slots[k] for k in honest], :P].astype(f64)
        assert AA.gamma_of(V, "minmax_" + attack.split("_")[1])[2] > 1.2, attack
        assert TA.craft(stack[:, :P].astype(f64), slots, honest, rule, H, attack, 3e38)[1] == 0
    a, b = torch.nan_to_num(dst, 7.0).cpu().numpy(), torch.nan_to_num(ref, 7.0).cpu().numpy()
    assert a.view(np.uint32).tolist() == b.view(np.uint32).tolist()
    assert (gam[:, 0] == 0).all()


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(5300)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])[1::5][:32]
    dst, gam, jobs = _launch(K, msgs, stack.shape[1], cases)
    assert len(jobs) == 32 and {c[1] for c in cases} == set(TA.RULES)

    def run(groups):
        dst.fill_(NAN)
        gam.fill_(NAN)
        for g in groups:
            K.ops.tailored_attack(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(gam, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_dst_and_gamma_untouched(K):
    rs = np.random.RandomState(5400)
    P = 700
    stack = _stack(rs, n_rows=8, P=P, n_bad=1)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((3, P), NAN, device=K.dev)
    gam = torch.full((3, 4), NAN, device=K.dev)
    J = K.ops.tailored_attack_job
    good = J(dst[0], msgs, P, P, [0, 1, -1, 2], [0, 1, 3], "gmed", 1, "tailored_std", 2.0, gamma_out=gam[0, :1])
    d, g = dst[1], gam[1, :1]
    big = torch.full((2, 19 * 1536 // 5 + 1), 1.0, device=K.dev)
    bad = [J(d, msgs, P, 0, [0, -1], [0], "clip", 0, "tailored_uv", 1.0, gamma_out=g),
           J(d, msgs, P, P, [], [], "clip", 0, "tailored_uv", 1.0, gamma_out=g),
           J(d, msgs, P, P, [0] * 16 + [-1], [0], "clip", 0, "tailored_uv", 1.0, gamma_out=g),    # 17 slots
           J(d, msgs, P, P, [0, 1, 2], [0, 1, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=g),    # no crafted slot
           J(d, msgs, P, P, [-1, -1, 2], [], "clip", 0, "tailored_uv", 1.0, gamma_out=g),         # no honest slot
           J(d, msgs, P, P, [0, -1, 2], [0, 1], "clip", 0, "tailored_uv", 1.0, gamma_out=g),      # crafted honest
           J(d, msgs, P, P, [0, -2, 2], [0], "clip", 0, "tailored_uv", 1.0, gamma_out=g),         # negative row
           J(d, msgs, P, P, [0, -1, 2], [0], (2, 0), 0, "tailored_uv", 1.0, gamma_out=g),         # unknown family
           J(d, msgs, P, P, [0, -1, 2], [0], (0, 3), 0, "tailored_uv", 1.0, gamma_out=g),         # unknown rule
           J(d, msgs, P, P, [0, -1, 2], [0], (1, 4), 0, "tailored_uv", 1.0, gamma_out=g),
           J(d, msgs, P, P, [0, -1, 2], [0], "clip", 0, 3, 1.0, gamma_out=g),                     # unknown dev
           J(d, msgs, P, P, [0, -1, 2], [0], "trim", 2, "tailored_uv", 1.0, gamma_out=g),         # 2H >= n_in
           J(d, msgs, P, P, [0, -1, 2, 3], [0, 2, 3], "krum", 2, "tailored_uv", 1.0, gamma_out=g),  # n_in < H + 3
           J(d, msgs, P, P, [0, -1, 2], [0], "wmsr", 3, "tailored_uv", 1.0, gamma_out=g),         # H >= n_in
           J(d, msgs, P, P, [0, -1, 2], [0], "clip", -1, "tailored_uv", 1.0, gamma_out=g),
           J(d, msgs, P, P, [0, -1, 2], [0], "clip", 0, "tailored_sgn", -0.5, gamma_out=g),
           J(d, msgs, P, P, [0, -1, 2], [0], "clip", 0, "tailored_sgn", NAN, gamma_out=g),
           J(d, msgs, P, P, [0, -1, 2], [0], "clip", 0, "tailored_sgn", float("inf"), gamma_out=g),
           J(d, big, big.shape[1], big.shape[1], [0, -1], [0], "clip", 0, "tailored_std", 1.0, gamma_out=g),  # bound
           J(msgs[2], msgs, P, P, [0, -1, 2], [0, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=g),  # dst on a real slot
           J(msgs[1][3:], msgs, P, P, [5, -1], [0], "clip", 0, "tailored_uv", 1.0, gamma_out=g),    # ... of the other job
           J(d, msgs, P, P, [4, -1, 5], [0, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=msgs[5][9:]),  # gamma_out on a row
           J(d, msgs, P, P, [4, -1, 5], [0, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=msgs[1][9:]),
           J(d, msgs, P, P, [4, -1, 5], [0, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=dst[0][10:]),
           J(d, msgs, P, P, [4, -1, 5], [0, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=gam[0]),
           J(dst[0][1:], msgs, P, P - 1, [4, -1, 5], [0, 2], "clip", 0, "tailored_uv", 1.0, gamma_out=g)]
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.tailored_attack([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(gam).all()
    with pytest.raises(K.L.RcmarlError):
        J(d, msgs, P, P, [0, -1], [0], "clip", 0, "minmax_uv", 1.0)
    with pytest.raises(K.L.RcmarlError):
        K.ops.tailored_attack([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(gam).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "a message row was written"
    K.ops.tailored_attack([good])
    assert torch.isfinite(dst[0]).all() and torch.isnan(dst[1:]).all() and float(gam[0, 0]) >= 0
    assert torch.isnan(gam[0, 1:]).all() and torch.isnan(gam[1:]).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import tailored_attack_oracle as TA
rs = np.random.RandomState(5500)
P = L.TAILORED_MAX_FLOATS // 19
assert 19 * P == L.TAILORED_MAX_FLOATS
X = (rs.randn(16, P) * rs.uniform(0.1, 1, size=(16, 1)) + rs.randn(P)).astype(np.float32)
msgs = torch.as_tensor(X).cuda()
dst = torch.full((2, P), float("nan"), device="cuda")
gam = torch.full((2,), float("nan"), device="cuda")
slots = list(range(15)) + [-1]
honest = list(range(15))
ops.tailored_attack([ops.tailored_attack_job(dst[0], msgs, P, P, slots, honest, "gmed", 3, "tailored_std", 2.0, gamma_out=gam[0:1]),
                     ops.tailored_attack_job(dst[1], msgs, P, P, slots, honest, "trim", 3, "tailored_uv", 2.0, gamma_out=gam[1:2])])
for j, (rule, attack) in enumerate((("gmed", "tailored_std"), ("trim", "tailored_uv"))):
    want, g, O = TA.craft(X.astype(np.float64), slots, honest, rule, 3, attack, 2.0)
    got_g = float(gam[j])
    i = int(np.argmax(O))
    if TA.margin(O) > 1e-4:
        assert abs(got_g - g) <= 5e-5 * max(g, 1e-30), (rule, got_g, g)
        err = float(np.abs(dst[j].cpu().numpy() - want).max())
        assert err <= 1e-4 * max(np.abs(X).max(), 1), (rule, err)
    assert np.isfinite(dst[j].cpu().numpy()).all()
print("ok")
"""


def test_staging_bound_as_the_first_launch_of_a_process(K, tmp_path):
    """Two jobs of (16 + 3) * 1536 floats, RCMARL_TAILORED_MAX_FLOATS (117 KB of dynamic shared memory), as the first
    tailored launch of a fresh process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=600,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
def _coop_agent(w, rule, gamma, H, fast):
    if rule in VO.RULES:
        return VO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, aggregation=rule)
    return AO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, aggregation=rule)


def _oracle_round(agents, labels, in_nodes, rows, attacks, rules, H, N, T, round_, seed=0, n_epochs=2):
    prs = np.random.RandomState(1700)
    used, gammas, objs = [], {}, {}

    def rec(T_):
        p = prs.permutation(T_)
        used.append(p)
        return p
    hook = TA.make_hook(labels, in_nodes, attacks, rules, H, seed=seed, round_=round_, gammas=gammas, objectives=objs)
    loss = AT.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=rec, messages_hook=hook)
    return loss, used, gammas, objs


def _check_gammas(tr, want, objs):
    got = tr.attack_gammas()
    assert sorted(got) == sorted(want)
    small = np.inf
    for k, g in got.items():
        assert g.dtype == np.float32 and g.shape == (2,)
        for t in range(2):
            if k in objs:
                m = TA.margin(objs[k][t])
                small = min(small, m)
                if m <= MARGIN:
                    continue
            close(g[t], want[k][t], rtol=2e-3, atol=1e-12, err_msg=f"pair {k} net {t}")
    print(f"smallest gamma margin {small:.3g}")


def _synth(rs, B, NA=5, nrow=5):
    from kernel_util import synth
    return synth(rs, B, NA, nrow)


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("rule", TA.RULES)
@pytest.mark.parametrize("attack", TA.ATTACKS)
def test_c2_update_round_with_a_tailored_attacker(K, attack, rule, N):
    """The benchmark's 5-agent team with agent 4 Byzantine on a tailored attack (s = 2) and every cooperative agent on
    `rule`: one update round of two epochs against the oracle's round; one tailored launch per epoch in place of the
    rcmarl_attack one; attack_gammas against the oracle's last epoch."""
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(5600 + N)
    rows = _synth(rs, T * N)
    agents = [_coop_agent(w[i], rule, gamma, 1, 0.01) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    want, used, gammas, objs = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: (attack, 2.0)}, [rule] * 5, 1, N, T,
                                             round_, seed=9)
    assert sorted(gammas) == [(4, 1), (4, 2), (4, 3)]
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=9, aggregation=rule)
    launches = []
    for att in ((attack, 2.0), ("alie", 1.0)):
        it = iter(list(used))
        tr = Trainer(attack=att, perm_source=lambda T_: next(it), **cfg)
        tr.load_rows(*rows)
        tr.episodes_done = round_
        got = tr.update_round()
        launches.append(tr.launches)
        if att[0] == attack:
            assert next(it, None) is None and tr.tailor_pairs == [0, 1, 2] and tr.adapt_pairs == []
            for k in ("critic_loss", "TR_loss", "actor_loss"):
                np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
            for i in range(5):
                TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
            _check_gammas(tr, gammas, objs)
        else:
            assert tr.attack_gammas() == {} and tr.att_gamma is None
    assert launches[0] == launches[1]                      # one launch per epoch, tailored or not


# 16 agents on the 10x10 grid: 8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy
B16 = ["Cooperative", "Byzantine", "Cooperative", "Malicious", "Cooperative", "Byzantine", "Cooperative", "Greedy",
       "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Malicious", "Byzantine", "Cooperative"]
ATT16 = {1: ("tailored_std", 2.0), 5: ("tailored_std", 2.0), 9: ("tailored_uv", 1.0), 11: ("alie", 1.0),
         14: ("tailored_sgn", 2.0)}
RULES16 = ["clip", "gmed", "trim", "scclip", "wmsr", "clip", "gmed", "trim"]


def test_16_agent_team_with_colluding_tailored_attackers(K):
    """Circulant in-neighbourhoods of 10; four tailored attackers (receivers hear several of them: colluding crafted
    slots) and one ALIE attacker, with Malicious and Greedy agents among the real slots; coordinate and vector rules
    mixed per agent.  More than 32 tailored jobs, so two launches per epoch."""
    from rcmarl import nets
    from rcmarl.trainer import Trainer
    rs = np.random.RandomState(5700)
    NA = 16
    in_nodes = [[(i + k) % NA for k in range(10)] for i in range(NA)]
    w = [[nets.glorot_uniform(32, 5, rs), nets.glorot_uniform(32, 1, rs), nets.glorot_uniform(48, 1, rs)] for _ in range(NA)]
    for i in range(NA):
        if B16[i] == "Malicious":
            w[i].append(nets.glorot_uniform(32, 1, rs))
    desired, H, fast = rs.randint(0, 10, size=(NA, 2)), [i % 3 for i in range(NA)], [0.01 + 0.001 * (i % 4) for i in range(NA)]
    coop = [i for i, l in enumerate(B16) if l == "Cooperative"]
    rules = ["clip"] * NA
    for q, i in enumerate(coop):
        rules[i] = RULES16[q]
    pairs = AT.byzantine_pairs(B16, in_nodes)
    n_tail = sum(1 for b, _, _ in pairs if ATT16[b][0] in TA.ATTACKS)
    assert 2 * n_tail > 32
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(B16):
        if lab == "Cooperative":
            agents.append(_coop_agent(w[i], rules[i], gamma, H[i], fast[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    want, used, gammas, objs = _oracle_round(agents, B16, in_nodes, rows, ATT16, rules, H, N, T, round_, seed=4)
    it = iter(list(used))
    cfg = dict(labels=B16, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma, H=H,
               fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=4,
               aggregation=rules)
    tr = Trainer(attack=[ATT16.get(i) for i in range(16)], perm_source=lambda T_: next(it), **cfg)
    assert len(tr.tailor_pairs) == n_tail
    tr.load_rows(*rows)
    tr.episodes_done = round_
    launches = tr.launches
    got = tr.update_round()
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({B16[i]}, {rules[i]})")
    _check_gammas(tr, gammas, objs)
    it = iter(list(used))
    tf = Trainer(labels=["Faulty" if l == "Byzantine" else l for l in B16],
                 **{k: v for k, v in cfg.items() if k != "labels"}, perm_source=lambda T_: next(it))
    tf.load_rows(*rows)
    tf.update_round()
    assert (tr.launches - launches) - tf.launches == 2 * 3      # two tailored and one ALIE launch per epoch


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


def test_world1_peer_comm_with_a_tailored_attacker_is_bitwise(K, gloo_world1):
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["gmed", "clip", "mkrum", "trim", "clip"], attack=("tailored_std", 2.0))
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append([getattr(tr, n).clone() for n in ("actor", "critic", "tr", "adam_m", "adam_v", "msg_c", "msg_t",
                                                       "att_gamma")])
    assert all(torch.equal(x, y) for x, y in zip(*runs))
