"""GPU parity of the dissensus and mimic attacks (rcmarl_dissensus_attack, rcmarl_mimic_attack, include/rcmarl.h)
against the float64 oracle (tests/dissensus_mimic_oracle.py): the kernels at n_honest 1..16 and the C2 / C3 parameter
counts in launches of 32 jobs, the bitwise consequences the header states, bitwise determinism, the refusals, and the
mimic staging bound in a fresh process; whole update rounds through Trainer (C2 with agent 4 Byzantine under the 8 rules
with and without nearest-neighbour mixing, the mimic state across rounds and through a checkpoint, a 16-agent team with
colluding attackers), a world-1 PeerComm and the drop-in train_RPBCAC path.

Tolerances: a dissensus message within 1e-6 (1 + c n) max|v| of the fp64 oracle (c = eps / n_byz, n summed
differences); the mimic direction within 1 - cos <= 1e-6 after Init and 1e-5 after a step; the copied row exactly
where the oracle's relative score margin exceeds 1e-4 (dissensus_mimic_oracle.pick_margin; identical rows tie exactly
and do not count), elsewhere within that margin of the best, and in update rounds the oracle follows the kernel's pick
there.  After whole update rounds weights rtol 1e-3 / atol 5e-5 and losses rtol 2e-3 / atol 2e-5 (as
test_trainer_gpu.py)."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import dissensus_mimic_oracle as DM                    # noqa: E402
import nnm_oracle as NO                                # noqa: E402
import team_util as TU                                 # noqa: E402
import test_nnm_gpu as NG                              # noqa: E402  (the C2 round helpers)
from golden_util import pretrained                     # noqa: E402
from kernel_util import close, load_kernels, synth, to_dev   # noqa: E402
from oracle import rpbcac_oracle as O                  # noqa: E402  (checker only)

f64 = np.float64
NAN = float("nan")
IN_NODES = NG.IN_NODES
C2_BYZ = NG.C2_BYZ
RULES = NG.RULES
WIDTHS = {"C2": (661, 761), "C3": (1101, 1421)}        # 5- / 16-agent critic, TR
PICK_GAP = 1e-4
INIT_GAP = 1e-4


@pytest.fixture(scope="module")
def K():
    return load_kernels()


def _stack(rs, n_rows=24, P=1421):
    centre = rs.randn(P)
    return (centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))).astype(np.float32)


def _cases(rs, n_rows=24):
    """(n_honest, P, honest rows, candidates) over n_honest 1..16 at both widths of C2 and C3: 64 jobs."""
    out = []
    for width in WIDTHS.values():
        for P in width:
            for n in range(1, 17):
                honest = [int(x) for x in rs.choice(n_rows, size=n, replace=False)]
                if n >= 4 and n % 3 == 1:
                    honest[-1] = honest[1]                                     # a repeated entry
                cand = DM.candidates(honest[0], honest)
                out.append((n, P, honest, cand))
    return out


# ---------------------------------------------------------------------------------------------------------- dissensus
def test_dissensus_against_the_oracle(K):
    rs = np.random.RandomState(6100)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    S = stack.shape[1]
    cases = _cases(rs)
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        dst = torch.full((len(part), S), NAN, device=K.dev)
        spec = []
        for j, (n, P, honest, _) in enumerate(part):
            n_byz, eps = int(rs.randint(1, 5)), float(rs.choice([0.5, 1.0, 2.5, 7.0]))
            spec.append((n_byz, eps))
        K.ops.dissensus_attack([K.ops.dissensus_attack_job(dst[j], msgs, S, P, h[0], h, *spec[j])
                                for j, (_, P, h, _) in enumerate(part)])
        got = dst.cpu().numpy()
        for j, (n, P, honest, _) in enumerate(part):
            n_byz, eps = spec[j]
            V = stack[honest, :P].astype(f64)
            want = DM.dissensus(V[0], V, n_byz, eps)
            c = eps / n_byz
            assert np.isnan(got[j, P:]).all()
            close(got[j, :P], want, rtol=0, atol=1e-6 * (1 + c * n) * np.abs(V).max(), err_msg=f"n={n} P={P}")


def test_dissensus_eps_zero_is_x_bitwise(K):
    rs = np.random.RandomState(6150)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    S = stack.shape[1]
    dst = torch.full((16, S), NAN, device=K.dev)
    jobs = [K.ops.dissensus_attack_job(dst[n - 1], msgs, S, S, 20 - n, list(range(n)), 1 + n % 3, 0.0)
            for n in range(1, 17)]
    K.ops.dissensus_attack(jobs)
    got = dst.cpu().numpy()
    for n in range(1, 17):
        np.testing.assert_array_equal(got[n - 1], stack[20 - n])


# ---------------------------------------------------------------------------------------------------------- mimic
def _mimic_launch(K, msgs, S, part, z, update, dst=None, tgt=None):
    dst = torch.full((len(part), S), NAN, device=K.dev) if dst is None else dst
    tgt = torch.full((len(part), 1), -7, dtype=torch.int32, device=K.dev) if tgt is None else tgt
    K.ops.mimic_attack([K.ops.mimic_attack_job(dst[j], msgs, S, P, h, c, z[j], update, target_out=tgt[j])
                        for j, (_, P, h, c) in enumerate(part)])
    return dst.cpu().numpy(), tgt.cpu().numpy()[:, 0]


def _cos(a, b):
    na, nb = np.linalg.norm(a), np.linalg.norm(b)
    return float(a.astype(f64) @ b.astype(f64) / (na * nb)) if na > 0 and nb > 0 else (1.0 if na == nb == 0 else 0.0)


def _check_pick(stack, part, j, got_k, got_dst, t, tag):
    n, P, honest, cand = part[j]
    V = stack[honest, :P].astype(f64)
    assert got_k in cand, tag
    np.testing.assert_array_equal(got_dst[j, :P], stack[honest[got_k], :P], err_msg=tag)   # a bitwise copy
    assert np.isnan(got_dst[j, P:]).all(), tag
    want = int(np.argmax(t)) if np.isfinite(t).any() else min(cand)
    if DM.pick_margin(V, t) > PICK_GAP:
        assert np.array_equal(V[got_k], V[want]), f"{tag}: copied {got_k}, oracle {want}"
        return 1
    assert t[got_k] >= t.max() - PICK_GAP * abs(t.max()), tag
    return 0


def test_mimic_against_the_oracle(K):
    """Init (update 0), then one step (update 1) from the Init direction, then Init and a step in one call, at n_honest
    1..16 and the C2 / C3 widths: z against the fp64 oracle by cosine, the pick exactly where the margin is clear."""
    rs = np.random.RandomState(6200)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    S = stack.shape[1]
    cases = _cases(rs)
    n_exact = n_picks = 0
    for g in range(0, len(cases), 32):
        part = cases[g:g + 32]
        z = torch.zeros(len(part), S, device=K.dev)
        dst, k = _mimic_launch(K, msgs, S, part, z, 0)
        z_init = z.cpu().numpy()
        z_one = torch.zeros(len(part), S, device=K.dev)
        dst1, k1 = _mimic_launch(K, msgs, S, part, z_one, 1)                   # Init and a step in one call
        dst2, k2 = _mimic_launch(K, msgs, S, part, z, 1)                       # a step from the Init direction
        z_step, z_one = z.cpu().numpy(), z_one.cpu().numpy()
        np.testing.assert_array_equal(z_step, z_one)
        np.testing.assert_array_equal(k1, k2)
        for j, (n, P, honest, cand) in enumerate(part):
            tag = f"n={n} P={P} honest={honest}"
            V = stack[honest, :P].astype(f64)
            assert (z_init[j, P:] == 0).all() and (z_step[j, P:] == 0).all(), tag
            # Init: the oracle follows the kernel's k0 only where the largest e_k is a near tie
            k0 = None
            if DM.init_margin(V) <= INIT_GAP and z_init[j].any():
                C = DM.centred(V)
                k0 = int(np.argmax([_cos(z_init[j, :P], c) for c in C]))
            kw, zw, tw = DM.mimic(V, cand, np.zeros(P), 0, k0=k0)
            assert 1 - _cos(z_init[j, :P], zw) <= 1e-6, tag
            n_exact += _check_pick(stack, part, j, int(k[j]), dst, tw, tag + " init")
            ks, zs, ts = DM.mimic(V, cand, z_init[j, :P].astype(f64), 1)
            assert 1 - _cos(z_step[j, :P], zs) <= 1e-5, tag
            n_exact += _check_pick(stack, part, j, int(k2[j]), dst2, ts, tag + " step")
            n_picks += 2
    print(f"mimic picks compared exactly {n_exact} of {n_picks}")
    assert n_exact >= 0.8 * n_picks


def test_mimic_bitwise_consequences(K):
    """update 0 keeps a non-zero z bitwise; equal honest rows keep z at 0 and copy the lowest candidate; an S_j of the
    receiver alone copies the receiver."""
    rs = np.random.RandomState(6300)
    S = 761
    stack = _stack(rs, P=S)
    stack[19] = np.round(stack[19] * 16) / 16           # a row whose sums of up to 16 copies are exact in fp32 ...
    stack[20:24] = stack[19]                             # ... repeated: rows 19 .. 23 are equal, and so is their mean
    msgs = to_dev(K, stack)[0]
    part = [(4, S, [3, 7, 9, 11], [1, 2, 3]), (3, 661, [19, 20, 21], [2, 1]), (1, S, [5], [0]),
            (5, S, [22, 19, 23, 20, 21], [4, 3]), (16, S, list(range(16)), [0, 5, 15])]
    z0 = torch.as_tensor(rs.randn(len(part), S).astype(np.float32), device=K.dev)
    z0[1:4] = 0
    z = z0.clone()
    dst, k = _mimic_launch(K, msgs, S, part, z, 0)
    assert torch.equal(z[0], z0[0]) and torch.equal(z[4], z0[4])              # update 0: unchanged
    assert not z[1:4].any()                                                    # equal rows / one row: z stays 0
    assert list(k[1:4]) == [1, 0, 3]                                           # the lowest candidate
    for j in range(1, 4):
        n, P, h, c = part[j]
        np.testing.assert_array_equal(dst[j, :P], stack[h[k[j]], :P])
    np.testing.assert_array_equal(dst[2], stack[5])
    z = z0.clone()
    _mimic_launch(K, msgs, S, part, z, 1)
    assert not z[1:4].any() and not torch.equal(z[0], z0[0])


def test_bitwise_deterministic_across_calls_orders_and_splits(K):
    rs = np.random.RandomState(6400)
    stack = _stack(rs)
    msgs = to_dev(K, stack)[0]
    S = stack.shape[1]
    cases = _cases(rs)[::2]
    assert len(cases) == 32
    dst = torch.full((32, S), NAN, device=K.dev)
    ddst = torch.full((32, S), NAN, device=K.dev)
    tgt = torch.full((32, 1), -7, dtype=torch.int32, device=K.dev)
    z = torch.zeros(32, S, device=K.dev)
    mj = [K.ops.mimic_attack_job(dst[j], msgs, S, P, h, c, z[j], 1, target_out=tgt[j]) for j, (_, P, h, c) in enumerate(cases)]
    dj = [K.ops.dissensus_attack_job(ddst[j], msgs, S, P, h[0], h, 1 + j % 3, 1.5) for j, (_, P, h, _) in enumerate(cases)]

    def run(order):
        for t in (dst, ddst):
            t.fill_(NAN)
        tgt.fill_(-7)
        z.zero_()
        for g in order:
            K.ops.mimic_attack([mj[i] for i in g])
            K.ops.dissensus_attack([dj[i] for i in g])
        K.ops.mimic_attack(mj)                                             # a second epoch from the new z
        return [torch.nan_to_num(t, 7.0).clone() for t in (dst, ddst, z)] + [tgt.clone()]
    idx = list(range(32))
    first = run([idx])
    for order in ([idx], [idx[::-1]], [idx[5:9], idx[:5], idx[9:]], [[i] for i in idx]):
        again = run(order)
        assert all(torch.equal(a, b) for a, b in zip(first, again))


def test_refusals_leave_every_output_untouched(K):
    rs = np.random.RandomState(6500)
    P = 700
    stack = _stack(rs, n_rows=8, P=P)
    msgs = to_dev(K, stack)[0]
    dst = torch.full((2, P), NAN, device=K.dev)
    z = torch.full((2, P), 3.0, device=K.dev)
    tgt = torch.full((2, 1), -7, dtype=torch.int32, device=K.dev)
    M, D = K.ops.mimic_attack_job, K.ops.dissensus_attack_job
    good = M(dst[0], msgs, P, P, [0, 1, 2], [1, 2], z[0], 1, target_out=tgt[0])
    bad = [M(dst[1], msgs, P, P, [0, 1, 2], [1], z[1], 2, target_out=tgt[1]),                 # update 2
           M(dst[1], msgs, P, P, [0, -1, 2], [1], z[1], 1),
           M(dst[1], msgs, P, P, list(range(8)) * 2 + [0], [1], z[1], 1),                       # 17 honest rows
           M(dst[1], msgs, P, 0, [0, 1, 2], [1], z[1], 1),
           M(dst[1], msgs, P, 19 * 1536 // 6 + 1, [0, 1, 2], [1], z[1], 1),                   # staging bound
           M(msgs[2], msgs, P, P, [0, 1, 2], [1], z[1], 1),                                    # dst on an honest row
           M(dst[1], msgs, P, P, [0, 1, 2], [1], msgs[1], 1),                                  # z on an honest row
           M(dst[1], msgs, P, P, [5, 6], [1], z[1], 1, target_out=msgs[0][3:]),                 # target on the other's
           M(dst[1], msgs, P, P, [5, 6], [1], z[0][100:], 1),                                  # z on the other's z
           M(dst[0][P // 2:], msgs, P, P, [5, 6], [1], z[1], 1),                               # dsts overlap
           M(dst[1], msgs, P, P, [5, 6], [1], z[1], 1, target_out=tgt[0])]                     # targets overlap
    for b in bad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.mimic_attack([good, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all() and (z == 3).all() and (tgt == -7).all()
    mask0 = M(dst[1], msgs, P, P, [5, 6], [1], z[1], 1)
    mask0.candidate_mask = 0
    for b in [mask0]:
        with pytest.raises(K.L.RcmarlError):
            K.ops.mimic_attack([good, b])
    with pytest.raises(K.L.RcmarlError):
        K.ops.mimic_attack([good] * 33)
    dgood = D(dst[0], msgs, P, P, 0, [0, 1, 2], 1, 1.0)
    dbad = [D(dst[1], msgs, P, P, 0, [0, 1, 2], 0, 1.0), D(dst[1], msgs, P, P, 0, [0, 1, 2], 1, -1.0),
            D(dst[1], msgs, P, P, 0, [0, 1, 2], 1, NAN), D(dst[1], msgs, P, P, -1, [0, 1, 2], 1, 1.0),
            D(msgs[7], msgs, P, P, 7, [4, 5], 1, 1.0),                                         # dst on its own row
            D(msgs[2], msgs, P, P, 4, [5, 6], 1, 1.0),                                         # ... the other's honest
            D(dst[0][10:], msgs, P, P, 4, [5, 6], 1, 1.0)]                                     # dsts overlap
    for b in dbad:
        with pytest.raises(K.L.RcmarlError):
            K.ops.dissensus_attack([dgood, b])
        torch.cuda.synchronize()
        assert torch.isnan(dst).all()
    assert np.array_equal(msgs.cpu().numpy(), stack), "an honest row was written"
    K.ops.mimic_attack([good])
    assert torch.isfinite(dst[0]).all() and torch.isnan(dst[1]).all() and int(tgt[0]) in (1, 2) and (z[1] == 3).all()


FRESH = r"""
import sys
sys.path[:0] = sys.argv[1:]
import numpy as np, torch
from rcmarl import _lib as L, ops
import dissensus_mimic_oracle as DM
rs = np.random.RandomState(6600)
P = L.MIMIC_MAX_FLOATS // 19
X = (rs.randn(16, P) * rs.uniform(0.1, 1, size=(16, 1)) + rs.randn(P)).astype(np.float32)
msgs = torch.as_tensor(X).cuda()
dst = torch.full((P,), float("nan"), device="cuda")
z = torch.zeros(P, device="cuda")
t = torch.full((1,), -1, dtype=torch.int32, device="cuda")
ops.mimic_attack([ops.mimic_attack_job(dst, msgs, P, P, list(range(16)), list(range(1, 16)), z, 1, target_out=t)])
k, zw, tw = DM.mimic(X.astype(np.float64), range(1, 16), np.zeros(P), 1)
zz = z.cpu().numpy().astype(np.float64)
assert 1 - zz @ zw / np.linalg.norm(zz) / np.linalg.norm(zw) <= 1e-5
assert DM.pick_margin(X.astype(np.float64), tw) <= 1e-4 or int(t) == k, (int(t), k)
assert np.array_equal(dst.cpu().numpy(), X[int(t)])
print("ok")
"""


def test_staging_bound_as_the_first_launch_of_a_process(K, tmp_path):
    """16 honest rows of 1536 parameters ((16 + 3) * 1536 = RCMARL_MIMIC_MAX_FLOATS, 114 KB of dynamic shared memory)
    as the first mimic launch of a fresh process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    paths = [os.path.join(root, "resilient-consensus-based-marl_b200"), os.path.join(root, "tests"), root]
    out = subprocess.run([sys.executable, "-s", "-c", FRESH, *paths], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---------------------------------------------------------------------------------------------------------- Trainer
def _targets(runs):
    return {e: tr.mimic_targets() for e, tr in enumerate(runs)}


def _oracle_round(agents, labels, in_nodes, rows, attacks, rules, mixing, H, N, T, round_, runs, kernel_M, seed,
                  n_epochs=2, hook=None):
    hook = hook or DM.StateHook(labels, in_nodes, attacks, rules, H, seed=seed, round_=round_, gap=PICK_GAP)
    hook.follow = _targets(runs)
    outer = hook
    if any(m is not None for m in mixing):
        outer = NO.mixing_hook(labels, in_nodes, mixing, H, inner=hook, kernel_M=kernel_M)
    loss = NO.update_round(agents, labels, in_nodes, *rows, n_envs=N, n_epochs=n_epochs, n_actor_steps=T,
                           common_reward=False, perm_source=NG._perms(), messages_hook=outer)
    return loss, hook


def _check_targets(tr, hook):
    got = tr.mimic_targets()
    assert sorted(got) == sorted(hook.targets)
    for key, k in got.items():
        for t in range(2):
            if hook.margins[key][t] > PICK_GAP:
                assert int(k[t]) == hook.targets[key][t], (key, t)
            else:
                assert int(k[t]) == hook.targets[key][t]                       # the oracle followed the kernel


ATTACKS = {"dissensus": 1.0, "mimic": 1}


@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("mixing", [None, "nnm"])
@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("kind", list(ATTACKS))
def test_c2_update_round_with_a_byzantine_agent(K, kind, rule, mixing, N):
    """The benchmark's 5-agent team with agent 4 Byzantine (H = 1), every cooperative agent on `rule`, with and without
    mixing: two epochs against the oracle's round with the state hook; one launch per epoch more than a Faulty agent
    4, and the message rows of any other attack.  mimic at T0 = 1: a step in epoch 0, the direction frozen in epoch 1."""
    w, desired, _ = pretrained()
    gamma, T, round_ = 0.9, 40, 150
    rs = np.random.RandomState(6700 + N)
    rows = synth(rs, T * N)
    attack = (kind, ATTACKS[kind])
    cfg = dict(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=N, gamma=gamma, H=1, fast_lr=0.01,
               slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=9, attack=attack, aggregation=rule)
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, mixing)
    agents = [NG._oracle_agent(rule, w[i], 0.01, gamma, 1) for i in range(4)]
    agents.append(O.FaultyOracleAgent(w[4][0], w[4][1], w[4][2], 0.002, gamma, dtype=f64))
    NG._follow_dnc(agents, runs)
    mix = [mixing] * 4 + [None]
    want, hook = _oracle_round(agents, C2_BYZ, IN_NODES, rows, {4: attack}, [rule] * 5, mix, [1] * 5, N, T, round_,
                               runs, kernel_M, seed=9)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(5):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i}")
    if kind == "mimic":
        _check_targets(tr, hook)
        assert tr.mimic_steps == [1, 1, 1] and tr.mimic_pairs == [0, 1, 2]
        assert "mimic_z" in tr.state_dict(include_buffer=False)
    else:
        assert tr.diss_pairs == [0, 1, 2] and "mimic_z" not in tr.state_dict(include_buffer=False)
    faulty, _ = NG._trainer_round(dict(cfg, labels=C2_BYZ[:4] + ["Faulty"], attack=None), rows, round_, 2, mixing)
    other, _ = NG._trainer_round(dict(cfg, attack=("alie", 1.0)), rows, round_, 2, mixing)
    assert tr.launches - faulty.launches == 2                                  # one launch per epoch
    assert tr.launches == other.launches and tr.msg_c.shape == other.msg_c.shape and tr.msg_t.shape == other.msg_t.shape


def _c2_trainer(T0, n_epochs=2, seed=31):
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    return Trainer(labels=C2_BYZ, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=16, gamma=0.9, H=1,
                   fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=n_epochs, buffer_size=100,
                   seed=seed, aggregation="mkrum", mixing="nnm", attack=("mimic", T0))


def _state(tr):
    return [getattr(tr, n).clone() for n in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v", "msg_c", "msg_t",
                                             "mimic_z", "mimic_target", "mix_weights")]


def test_mimic_state_carries_over_rounds_and_checkpoints(K, tmp_path):
    """Two rounds carry z over (the second round starts from the first's z, not from Init); saving after the first
    round, loading into a fresh trainer and continuing is bitwise equal to continuing; after T0 steps z is frozen."""
    a = _c2_trainer(3)
    a.rollout_block()
    a.update_round()
    assert a.mimic_steps == [2, 2, 2]
    z1 = a.mimic_z.clone()
    assert z1[:, 0, :a.PC].abs().sum(1).gt(0).all() and not z1[:, 0, a.PC:].any()
    a.save(tmp_path / "ckpt.pt")
    b = _c2_trainer(3)
    b.load(tmp_path / "ckpt.pt")
    assert torch.equal(b.mimic_z, z1) and b.mimic_steps == [2, 2, 2]
    fresh = _c2_trainer(3)                                 # the same round without the carried state
    fresh.load_state_dict({k: v for k, v in a.state_dict().items() if k not in ("mimic_z", "mimic_steps")}
                          | dict(mimic_z=torch.zeros_like(z1).cpu(), mimic_steps=[0, 0, 0]))
    for tr in (a, b, fresh):
        tr.rollout_block()
        tr.update_round()
    assert a.mimic_steps == b.mimic_steps == [3, 3, 3]
    assert all(torch.equal(x, y) for x, y in zip(_state(a), _state(b)))
    assert not torch.equal(a.mimic_z, fresh.mimic_z)      # the carried z mattered
    # frozen after T0: a one-epoch and a three-epoch round from the same state end with the same z
    ends = []
    for n_epochs in (1, 3):
        tr = _c2_trainer(1, n_epochs=n_epochs)
        tr.rollout_block()
        tr.update_round()
        assert tr.mimic_steps == [1, 1, 1]
        ends.append(tr.mimic_z.clone())
    assert torch.equal(ends[0], ends[1])


def test_16_agent_team_with_colluding_attackers(K):
    """16 agents (8 cooperative, 5 Byzantine, 2 Malicious, 1 Greedy; in-neighbourhoods of 8, receiver 0 listing agent 1
    twice): agents 1, 5 and 14 mimic with the same T0, agents 9 and 11 run dissensus, so receivers hear two dissensus
    attackers (n_byz = 2) and two colluding mimic attackers.  The colluders' states and copies are bitwise equal, and the
    round matches the oracle's."""
    import test_attacks_gpu as TA
    rs = np.random.RandomState(2300)
    in_nodes, w, desired, H, fast, _ = TA._team16(rs)
    attacks = {1: ("mimic", 2), 5: ("mimic", 2), 14: ("mimic", 2), 9: ("dissensus", 1.0), 11: ("dissensus", 2.0)}
    labels = TA.B16
    gamma, T, N, round_ = 0.9, 40, 4, 7
    agents = TU.oracle_agents(labels, w, H, fast, gamma)
    rows = TU.grid_rows(rs, T * N, 16, 10)
    cfg = dict(labels=labels, in_nodes=in_nodes, weights=w, desired=desired, n_envs=N, nrow=10, ncol=10, gamma=gamma,
               H=H, fast_lr=fast, slow_lr=0.002, max_ep_len=10, n_ep_fixed=4, buffer_size=1000, seed=4,
               attack=[attacks.get(i) for i in range(16)])
    tr, got, kernel_M, runs = NG._kernel_M(cfg, rows, round_, None)
    want, hook = _oracle_round(agents, labels, in_nodes, rows, attacks, ["clip"] * 16, [None] * 16, H, N, T, round_,
                               runs, kernel_M, seed=4)
    for k in ("critic_loss", "TR_loss", "actor_loss"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, atol=2e-5, err_msg=k)
    for i in range(16):
        TU.close_w(tr.get_weights(i), agents[i].get_parameters(), msg=f"agent {i} ({labels[i]})")
    _check_targets(tr, hook)
    targets = tr.mimic_targets()
    pairs = [tr.byz_pairs[e][:2] for e in tr.mimic_pairs]
    by_recv = {}
    for q, (b, j) in enumerate(pairs):
        by_recv.setdefault(j, []).append(q)
    colluding = [qs for qs in by_recv.values() if len(qs) > 1]
    assert colluding, by_recv
    for qs in colluding:
        for q in qs[1:]:
            assert torch.equal(tr.mimic_z[q], tr.mimic_z[qs[0]])
            assert np.array_equal(targets[pairs[q]], targets[pairs[qs[0]]])
            e0, e1 = tr.mimic_pairs[qs[0]], tr.mimic_pairs[q]
            assert torch.equal(tr.msg_c[16 + e0], tr.msg_c[16 + e1]) and torch.equal(tr.msg_t[16 + e0], tr.msg_t[16 + e1])
    n_byz = {j: sum(i in (9, 11) for i in in_nodes[j]) for j in range(16) if labels[j] == "Cooperative"}
    assert max(n_byz.values()) == 2


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


def test_world1_peer_comm_with_the_new_attacks_is_bitwise(K, gloo_world1):
    """The peer-memory exchange of a one-rank world changes no bit of a run with a dissensus and a mimic attacker."""
    from rcmarl.comm import PeerComm
    from rcmarl.trainer import Trainer
    w, desired, _ = pretrained()
    labels = ["Cooperative", "Cooperative", "Byzantine", "Cooperative", "Byzantine"]
    runs = []
    for bound in (False, True):
        tr = Trainer(labels=labels, in_nodes=IN_NODES, weights=w, desired=desired, n_envs=64, gamma=0.9, H=1,
                     fast_lr=0.01, slow_lr=0.002, max_ep_len=8, n_ep_fixed=5, n_epochs=2, buffer_size=100, seed=21,
                     aggregation=["trim", "scclip", "clip", "dnc", "clip"], mixing=["nnm", None, None, "nnm", None],
                     attack=[None, None, ("dissensus", 2.0), None, ("mimic", 3)])
        if bound:
            tr.comm = PeerComm(0, 1)
            gloo_world1.append(tr.comm)
        for _ in range(2):
            tr.rollout_block()
            tr.update_round()
        torch.cuda.synchronize()
        runs.append([getattr(tr, n).clone() for n in ("actor", "critic", "tr", "adam_m", "adam_v", "msg_c", "msg_t",
                                                      "mimic_z", "mimic_target")])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_train_rpbcac_with_a_mimic_agent(K):
    """Drop-in path: train_RPBCAC with a Byzantine_CAC_agent(attack=("mimic", T0)) among the reference agents runs the
    mimic attack (one launch per epoch), and the same objects through a Trainer built directly give the same weights."""
    import contextlib
    import io
    from rcmarl import api
    import training.train_agents as training
    from agents.adversarial_CAC_agents import Byzantine_CAC_agent
    w, desired, _ = pretrained()
    labels = ["Cooperative"] * 4 + ["Byzantine"]
    cfg = dict(labels=["Cooperative"] * 4 + ["Faulty"], in_nodes=IN_NODES, weights=w, desired=desired, nrow=5, ncol=5,
               H=1, n_envs=8, gamma=0.9, fast_lr=0.01, slow_lr=0.002, max_ep_len=6, n_ep_fixed=4, n_epochs=2,
               buffer_size=48)
    env, agents, args = api.build_reference_objects(cfg)
    f = agents[4]
    agents[4] = Byzantine_CAC_agent(f.actor, f.critic, f.TR, slow_lr=0.002, gamma=0.9, attack=("mimic", 3))
    args["agent_label"] = labels
    args["n_episodes"] = 8
    with pytest.raises(K.L.RcmarlError):
        Byzantine_CAC_agent(f.actor, f.critic, f.TR, slow_lr=0.002, gamma=0.9, attack=("mimic", 2.5))
    with contextlib.redirect_stdout(io.StringIO()):
        weights, sim_data = training.train_RPBCAC(env, agents, args)
    tr = training.train_RPBCAC.last_trainer
    assert tr.mimic_pairs == [0, 1, 2] and tr.mimic_steps == [3, 3, 3]         # 2 rounds x 2 epochs, T0 = 3
    for (b, j), k in tr.mimic_targets().items():
        assert b == 4 and all(int(x) in IN_NODES[j] and int(x) != j for x in k)
    assert np.isfinite(sim_data.to_numpy()).all()
