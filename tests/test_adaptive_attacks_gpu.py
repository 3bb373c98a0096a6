"""GPU parity of the min-max / min-sum Byzantine messages (rcmarl_adaptive_attack, include/rcmarl.h) against the fp64
oracle (tests/adaptive_attack_oracle.py): the kernel for both kinds x three directions, n_honest 1..16 with repeated
indices, the trainer's parameter counts, 32 jobs per launch with gamma_out; scale 0 against rcmarl_attack's ALIE at
z = 0 bit for bit; bitwise determinism; a job at the staging bound as the first launch of a fresh process; the refusals;
whole update rounds through Trainer (the C2 team with agent 4 Byzantine under every attack and every rule, a 16-agent
team with several attackers, a world-1 PeerComm) and Trainer.attack_gammas.

Tolerances.  The kernel's distances are fp32 sums of up to 1421 squares (lane partials of 45 terms and a 5-level
butterfly: about 50 * 2^-24 = 3e-6 relative at worst), and gamma is a smooth function of them away from ties of the
minimum over k; on this file's data the fp32 oracle's gamma is within 2.4e-7 of the fp64 one.  gamma is compared with rtol
5e-5, and the message with atol 1e-5 max(|v|, 1) (the fp32 mean of at most 16 rows) plus 5e-5 gamma max|d| (gamma's
tolerance carried along d).  After whole update rounds the honest messages themselves carry the round's fp32 error:
weights rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as test_trainer_gpu.py), gamma rtol 2e-3.

Krum and multi-Krum select messages, and min-max puts the crafted one at the edge of the honest spread by construction.
So every selection the oracle makes in these rounds is checked for a relative score margin above 1e-4 (or exactly 0: a
tie in fp64 that the fp32 scores share, both breaking it to the lower index), as test_vector_rules_gpu.py does; a near
tie fails loudly instead of flaking.  With the data seeds 4300 + N the smallest non-zero margin of those rounds is 9.5e-3
(minsum_uv under mkrum at N = 1; the per-case minimum is printed).  Krum's selections (m = 1 of n = 4 at H = 1) are all
exact ties: the two closest messages share their score, D_kl, and both sides pick the lower index."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import adaptive_attack_oracle as AA                     # noqa: E402
import agg_oracle as AO                                 # noqa: E402
import attack_oracle as AT                              # noqa: E402
import team_util as TU                                  # noqa: E402
import vector_oracle as VO                              # noqa: E402
from golden_util import pretrained                      # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                   # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
C2_BYZ = ["Cooperative"] * 4 + ["Byzantine"]
PAR_COUNTS = (661, 761, 1101, 1421)                    # 5- / 16-agent critic / TR nets
RULES = ("clip", "trim", "wmsr") + VO.RULES
MARGIN = 1e-4
G_RTOL = 5e-5


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def msg_atol(vmax, g, dmax):
    return 1e-5 * max(vmax, 1.0) + G_RTOL * g * dmax


# ---------------------------------------------------------------------------------------------------------- kernel
def _stack(rs, n_rows=24, P=max(PAR_COUNTS)):
    """Messages around a common centre (as trained networks are), each row with its own spread."""
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def _cases(rs, n_rows):
    """(attack, honest, P) for every attack x n_honest 1..16, repeated indices in every third job"""
    out = []
    for a, attack in enumerate(AA.ATTACKS):
        for nh in range(1, 17):
            honest = [int(x) for x in rs.choice(n_rows, size=nh, replace=False)]
            if nh >= 3 and (nh + a) % 3 == 0:
                honest[-1] = honest[int(rs.randint(0, nh - 1))]
            out.append((attack, honest, PAR_COUNTS[(nh + a) % 4]))
    return out


def _launch(K, msgs, stride, cases, scale=1.0):
    dst = torch.full((len(cases), stride), NAN, device=K.dev)
    gam = torch.full((len(cases), 2), NAN, device=K.dev)
    jobs = [K.ops.adaptive_attack_job(dst[j], msgs, stride, P, honest, attack, scale, gamma_out=gam[j, :1])
            for j, (attack, honest, P) in enumerate(cases)]
    return dst, gam, jobs


def test_adaptive_attack_against_the_oracle(K):
    """Both kinds x three directions at every n_honest, the trainer's parameter counts, repeated honest indices; launches
    of exactly 32 jobs; the message and gamma_out against the fp64 oracle."""
    rs = np.random.RandomState(4100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])
    assert len(cases) == 96
    worst_g, worst_m, n_pos = 0.0, 0.0, 0
    for g0 in range(0, len(cases), 32):
        part = cases[g0:g0 + 32]
        dst, gam, jobs = _launch(K, msgs, stack.shape[1], part)
        K.ops.adaptive_attack(jobs)
        got, gg = dst.cpu().numpy(), gam.cpu().numpy()
        for j, (attack, honest, P) in enumerate(part):
            V = stack[honest, :P].astype(f64)
            want, g = AA.craft(V, attack, 1.0)
            d = AA.gamma_of(V, attack)[1]
            tag = f"{attack} n_honest={len(honest)} P={P} honest={honest}"
            assert np.isnan(got[j, P:]).all() and np.isnan(gg[j, 1]), f"{tag}: wrote past n / gamma_out"
            if len(set(honest)) == 1:
                assert gg[j, 0] == 0 and np.array_equal(got[j, :P], stack[honest[0], :P]), tag
                continue
            n_pos += g > 0
            close(gg[j, 0], g, rtol=G_RTOL, atol=0, err_msg=tag)
            atol = msg_atol(np.abs(V).max(), g, np.abs(d).max())
            close(got[j, :P], want, rtol=0, atol=atol, err_msg=tag)
            worst_g = max(worst_g, abs(gg[j, 0] - g) / g)
            worst_m = max(worst_m, np.abs(got[j, :P] - want).max() / atol)
    print(f"gamma > 0 in {n_pos} jobs; largest relative gamma error {worst_g:.2e}, largest message error "
          f"{worst_m:.3f} x atol")
    assert n_pos == 90                                   # every job with two distinct honest rows


def test_scale_zero_is_alie_at_z_zero_bitwise(K):
    """s = 0 writes the honest mean exactly as rcmarl_attack's ALIE at z = 0 does, and still reports gamma."""
    rs = np.random.RandomState(4150)
    stack = _stack(rs)
    stack[3, :50] = 0.0
    stack[7, 20:80] = -0.0
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])[::3]
    dst, gam, jobs = _launch(K, msgs, stack.shape[1], cases, scale=0.0)
    K.ops.adaptive_attack(jobs)
    ref = torch.full_like(dst, NAN)
    K.ops.attack([K.ops.attack_job(ref[j], msgs, stack.shape[1], P, honest, "alie", 0.0)
                  for j, (_, honest, P) in enumerate(cases)])
    d1, g1, jobs1 = _launch(K, msgs, stack.shape[1], cases, scale=1.0)
    K.ops.adaptive_attack(jobs1)
    torch.cuda.synchronize()
    a, b = torch.nan_to_num(dst, 7.0).cpu().numpy(), torch.nan_to_num(ref, 7.0).cpu().numpy()
    assert a.view(np.uint32).tolist() == b.view(np.uint32).tolist()
    assert torch.equal(torch.nan_to_num(gam, 7.0), torch.nan_to_num(g1, 7.0)) and bool((gam[:, 0] > 0).any())


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(4200)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    cases = _cases(rs, stack.shape[0])[1::3]
    dst, gam, jobs = _launch(K, msgs, stack.shape[1], cases)
    assert len(jobs) == 32 and {c[0] for c in cases} == set(AA.ATTACKS)

    def run(groups):
        dst.fill_(NAN)
        gam.fill_(NAN)
        for g in groups:
            K.ops.adaptive_attack(g)
        return torch.nan_to_num(dst, 7.0).clone(), torch.nan_to_num(gam, 7.0).clone()
    first = run([jobs])
    for groups in ([jobs], [jobs[::-1]], [jobs[5:9], jobs[:5], jobs[9:]], [[j] for j in jobs]):
        again = run(groups)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_refusals_leave_dst_and_gamma_untouched(K):
    rs = np.random.RandomState(4300)
    P = 700
    stack = _stack(rs, n_rows=8, P=P)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((3, P), NAN, device=K.dev)
    gam = torch.full((3, 4), NAN, device=K.dev)
    J = K.ops.adaptive_attack_job
    good = J(dst[0], msgs, P, P, [0, 1, 2, 3], "minmax_std", 1.0, gamma_out=gam[0, :1])
    d, g = dst[1], gam[1, :1]
    big = torch.full((2, 18 * 1536 // 3 + 1), 1.0, device=K.dev)
    bad = [J(d, msgs, P, 0, [0, 1], "minmax_uv", 1.0, gamma_out=g),
           J(d, msgs, P, P, [], "minmax_uv", 1.0, gamma_out=g),
           J(d, msgs, P, P, list(range(8)) * 2 + [0], "minsum_std", 1.0, gamma_out=g),       # 17 honest rows
           J(d, msgs, P, P, [0, -1], "minsum_std", 1.0, gamma_out=g),
           J(d, msgs, P, P, [0, 1], (2, 0), 1.0, gamma_out=g),                               # unknown kind
           J(d, msgs, P, P, [0, 1], (0, 3), 1.0, gamma_out=g),                               # unknown dev
           J(d, msgs, P, P, [0, 1], "minmax_sgn", -0.5, gamma_out=g),
           J(d, msgs, P, P, [0, 1], "minmax_sgn", NAN, gamma_out=g),
           J(d, msgs, P, P, [0, 1], "minmax_sgn", float("inf"), gamma_out=g),
           J(d, big, big.shape[1], big.shape[1], [0], "minmax_std", 1.0, gamma_out=g),       # 3 n over the bound
           J(msgs[2], msgs, P, P, [0, 1, 2], "minsum_uv", 1.0, gamma_out=g),                 # dst is an honest row
           J(msgs[3][3:], msgs, P, P, [5, 6], "minsum_uv", 1.0, gamma_out=g),                # ... of the other job
           J(d, msgs, P, P, [4, 5], "minsum_uv", 1.0, gamma_out=msgs[5][9:]),               # gamma_out on a row
           J(d, msgs, P, P, [4, 5], "minsum_uv", 1.0, gamma_out=msgs[1][9:]),               # ... of the other job
           J(d, msgs, P, P, [4, 5], "minsum_uv", 1.0, gamma_out=dst[0][10:]),               # ... on the other dst
           J(d, msgs, P, P, [4, 5], "minsum_uv", 1.0, gamma_out=gam[0]),                    # ... on its gamma_out
           J(dst[0][1:], msgs, P, P - 1, [4, 5], "minsum_uv", 1.0, gamma_out=g)]            # two dsts overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.adaptive_attack([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and torch.isnan(gam).all()
    with pytest.raises(K.L.RcmarlError):
        J(d, msgs, P, P, [0, 1], "alie", 1.0)
    with pytest.raises(K.L.RcmarlError):
        K.ops.adaptive_attack([good] * 33)
    torch.cuda.synchronize()
    assert torch.isnan(dst).all() and torch.isnan(gam).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an honest row was written"
    K.ops.adaptive_attack([good])
    assert torch.isfinite(dst[0]).all() and torch.isnan(dst[1:]).all() and float(gam[0, 0]) > 0
    assert torch.isnan(gam[0, 1:]).all() and torch.isnan(gam[1:]).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import adaptive_attack_oracle as AA
rs = np.random.RandomState(4400)
P = L.ADAPTIVE_MAX_FLOATS // 18
assert 18 * P == L.ADAPTIVE_MAX_FLOATS
X = (rs.randn(16, P) * rs.uniform(0.1, 1, size=(16, 1)) + rs.randn(P)).astype(np.float32)
msgs = torch.as_tensor(X).cuda()
dst = torch.full((2, P), float("nan"), device="cuda")
gam = torch.full((2,), float("nan"), device="cuda")
ops.adaptive_attack([ops.adaptive_attack_job(dst[0], msgs, P, P, list(range(16)), "minmax_std", 1.0, gamma_out=gam[0:1]),
                     ops.adaptive_attack_job(dst[1], msgs, P, P, list(range(16)), "minsum_uv", 1.0, gamma_out=gam[1:2])])
for j, attack in enumerate(("minmax_std", "minsum_uv")):
    want, g = AA.craft(X.astype(np.float64), attack, 1.0)
    d = AA.gamma_of(X.astype(np.float64), attack)[1]
    got_g = float(gam[j])
    assert abs(got_g - g) <= 5e-5 * g, (attack, got_g, g)
    err = float(np.abs(dst[j].cpu().numpy() - want).max())
    assert err <= 1e-5 * max(np.abs(X).max(), 1) + 5e-5 * g * np.abs(d).max(), (attack, err)
print("ok")
"""


def test_staging_bound_as_the_first_launch_of_a_process(K, tmp_path):
    """Two jobs of (16 + 2) * 1536 floats, RCMARL_ADAPTIVE_MAX_FLOATS (108 KB of dynamic shared memory), as the first
    adaptive launch of a fresh process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
class _MarginAgent(VO.RPBCACOracleAgent):
    """The vector oracle agent, recording the relative Krum score margin of every selection it makes."""

    def _aggregate(self, w, msgs):
        if self.aggregation in ("krum", "mkrum"):
            X = np.stack([AT.pack(m, self.dtype) for m in msgs])
            m = 1 if self.aggregation == "krum" else X.shape[0] - self.H
            s = np.sort(VO.krum_scores(X, self.H))
            margin = np.inf if m == X.shape[0] else (s[m] - s[m - 1]) / max(s[m], 1e-300)
            self.__dict__.setdefault("margins", []).append(margin)
        return super()._aggregate(w, msgs)


def _coop_agent(w, rule, gamma, H, fast):
    if rule in VO.RULES:
        return _MarginAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, aggregation=rule)
    return AO.RPBCACOracleAgent(w[0], w[1], w[2], 0.002, fast, gamma, H=H, dtype=f64, aggregation=rule)


def _oracle_round(agents, labels, in_nodes, rows, attacks, N, T, round_, seed=0, n_epochs=2):
    prs = np.random.RandomState(1700)
    used, gammas = [], {}

    def rec(T_):
        p = prs.permutation(T_)
        used.append(p)
        return p
    hook = AA.make_hook(labels, in_nodes, attacks, seed=seed, round_=round_, gammas=gammas)
    loss = AT.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=rec, messages_hook=hook)
    return loss, used, gammas


def _check_margins(agents):
    margins = [m for ag in agents for m in getattr(ag, "margins", [])]
    finite = [m for m in margins if np.isfinite(m)]
    bad = [m for m in finite if 0 < m <= MARGIN]
    print(f"{len(margins)} Krum selections; smallest non-zero relative margin "
          f"{min([m for m in finite if m > 0], default=np.inf):.3g}")
    assert not bad, f"near ties in the oracle's Krum selections: {bad}"


def _check_gammas(tr, want):
    got = tr.attack_gammas()
    assert sorted(got) == sorted(want)
    for k, g in got.items():
        assert g.dtype == np.float32 and g.shape == (2,)
        close(g, want[k], rtol=2e-3, atol=0, err_msg=f"pair {k}")


CASES = sorted({(a, "clip") for a in AA.ATTACKS} | {(a, r) for a in ("minmax_std", "minsum_uv") for r in RULES})


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("attack,rule", CASES)
def test_c2_update_round_with_an_adaptive_attacker(K, attack, rule, N):
    """The benchmark's 5-agent team with agent 4 Byzantine on an adaptive attack (s = 1) and every cooperative agent on
    `rule`: one update round of two epochs against the oracle's round with the per-receiver hook; one adaptive launch per
    epoch in place of the rcmarl_attack one; attack_gammas against the oracle's last epoch."""
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(4300 + N)
    rows = synth(rs, T * N)
    agents = [_coop_agent(w[i], rule, gamma, 1, 0.01) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    want, used, gammas = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: (attack, 1.0)}, N, T, round_, seed=9)
    _check_margins(agents)
    assert sorted(gammas) == [(4, 1), (4, 2), (4, 3)] and min(min(g) for g in gammas.values()) > 0
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=9, aggregation=rule)
    launches = []
    for att in ((attack, 1.0), ("alie", 1.0)):
        it = iter(list(used))
        tr = Trainer(attack=att, perm_source=lambda T_: next(it), **cfg)
        tr.load_rows(*rows)
        tr.episodes_done = round_
        got = tr.update_round()
        launches.append(tr.launches)
        if att[0] == attack:
            assert next(it, None) is None
            for k in ("critic_loss", "TR_loss", "actor_loss"):
                np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
            for i in range(5):
                TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
            _check_gammas(tr, gammas)
        else:
            assert tr.attack_gammas() == {} and tr.att_gamma is None
    assert launches[0] == launches[1]                      # one launch per epoch, adaptive or not


# 16 agents on the 10x10 grid (test_attacks_gpu.py's labels): 8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy
B16 = ["Cooperative", "Byzantine", "Cooperative", "Malicious", "Cooperative", "Byzantine", "Cooperative", "Greedy",
       "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Malicious", "Byzantine", "Cooperative"]
ATT16 = {1: ("minmax_std", 1.0), 5: ("minmax_std", 1.0), 9: ("minsum_uv", 1.0), 11: ("alie", 1.0),
         14: ("minsum_sgn", 0.5)}
RULES16 = ["clip", "gmed", "trim", "scclip", "wmsr", "clip", "gmed", "trim"]   # the 8 cooperative agents, in order


def test_16_agent_team_with_several_adaptive_attackers(K):
    """Circulant in-neighbourhoods of 10; four adaptive attackers and one ALIE attacker; coordinate and continuous vector
    rules mixed per agent.  More than 32 adaptive jobs, so two launches per epoch; receiver 0 hears agents 1 and 5, whose
    min-max messages for it are the same message (they see the same honest set) and must be bitwise equal."""
    from rcmarl import nets
    from rcmarl.trainer import Trainer
    rs = np.random.RandomState(4500)
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
    n_ada = sum(1 for b, _, _ in pairs if ATT16[b][0] in AA.ATTACKS)
    assert 2 * n_ada > 32 and 2 * (len(pairs) - n_ada) <= 32 and (1, 0, [0, 2, 4, 6, 8]) in pairs and (5, 0, [0, 2, 4, 6, 8]) in pairs
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = []
    for i, lab in enumerate(B16):
        if lab == "Cooperative":
            agents.append(_coop_agent(w[i], rules[i], gamma, H[i], fast[i]))
        else:
            agents.extend(TU.oracle_agents([lab], [w[i]], [H[i]], [fast[i]], gamma))
    rows = TU.grid_rows(rs, T * N, 16, 10)
    want, used, gammas = _oracle_round(agents, B16, in_nodes, rows, ATT16, N, T, round_, seed=4)
    it = iter(list(used))
    cfg = dict(labels=B16, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma, H=H,
               fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=1000, seed=4,
               aggregation=rules)
    tr = Trainer(attack=[ATT16.get(i) for i in range(16)], perm_source=lambda T_: next(it), **cfg)
    assert len(tr.adapt_pairs) == n_ada
    tr.load_rows(*rows)
    tr.episodes_done = round_
    launches = tr.launches
    got = tr.update_round()
    assert next(it, None) is None
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({B16[i]}, {rules[i]})")
    _check_gammas(tr, gammas)
    e1, e5 = [e for e, (b, j, _) in enumerate(tr.byz_pairs) if j == 0 and b in (1, 5)]
    for msgs in (tr.msg_c, tr.msg_t):
        assert torch.equal(msgs[NA + e1], msgs[NA + e5])
    g = tr.attack_gammas()
    assert np.array_equal(g[(1, 0)], g[(5, 0)])
    # with the attackers Faulty, the round makes two adaptive launches and one ALIE launch per epoch fewer
    it = iter(list(used))
    tf = Trainer(labels=["Faulty" if l == "Byzantine" else l for l in B16],
                 **{k: v for k, v in cfg.items() if k != "labels"}, perm_source=lambda T_: next(it))
    tf.load_rows(*rows)
    tf.update_round()
    assert (tr.launches - launches) - tf.launches == 2 * 3


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


def test_world1_peer_comm_with_an_adaptive_attacker_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run with a min-max attacker, gammas included."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["gmed", "clip", "mkrum", "trim", "clip"], attack=("minmax_std", 1.0))
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
    assert bool((runs[0][-1] > 0).all())
