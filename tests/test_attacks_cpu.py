"""CPU checks of the Byzantine attacks (rcmarl_attack, include/rcmarl.h): the NumPy Philox restatement against the
Random123 known-answer vectors, identities of the oracle's attacks, the oracle's update round with and without a
messages hook, the C layout of rcmarl_attack_job, and the refusals of the library and of Trainer before any device
work."""
import copy
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import attack_oracle as AT
import team_util as TU
from oracle import rpbcac_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIN = st.floats(-1e3, 1e3, allow_nan=False, width=64)


def hexwords(ws):
    return " ".join("%08x" % int(np.asarray(w).reshape(-1)[0]) for w in ws)


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    assert hexwords(AT.philox4x32_10(ctr, key)) == want


def test_counter_layout_and_box_muller():
    c = AT.counter(3, attacker=4, receiver=2, round_=150, epoch=7)
    assert [int(w[2]) for w in c] == [2, 0x40000204, 150, 7]
    x, y, _, _ = AT.philox4x32_10([w[1] for w in c], (5, 0))
    xi = AT.gauss_xi(3, 5, 4, 2, 150, 7)[1]
    u1, u2 = ((int(x) >> 8) + 1) / 2 ** 24, (int(y) >> 8) / 2 ** 24
    assert xi == np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2)
    big = AT.gauss_xi(200000, 11, 1, 3, 0, 0)
    assert abs(big.mean()) < 0.01 and abs(big.std() - 1) < 0.01 and np.isfinite(big).all()


@st.composite
def honest_sets(draw):
    n = draw(st.integers(1, 16))
    P = draw(st.integers(1, 5))
    return np.array(draw(st.lists(FIN, min_size=n * P, max_size=n * P)), np.float64).reshape(n, P)


@given(honest_sets())
@settings(max_examples=200, deadline=None)
def test_neutral_parameters_give_the_mean(v):
    mu = AT.moments(v)[0]
    xi = AT.gauss_xi(v.shape[1], 3, 4, 0, 0, 0)
    for got in (AT.craft(v, "alie", 0.0), AT.craft(v, "ipm", -1.0), AT.craft(v, "gauss", 0.0, xi)):
        np.testing.assert_array_equal(got, mu)
    np.testing.assert_allclose(mu, v.mean(0), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(AT.moments(v)[1], v.std(0), rtol=1e-9, atol=1e-9)


@given(st.lists(FIN, min_size=1, max_size=5), st.floats(-10, 10))
@settings(max_examples=100, deadline=None)
def test_alie_against_one_honest_message_sends_it(row, z):
    v = np.array([row])
    np.testing.assert_array_equal(AT.craft(v, "alie", z), v[0])


@given(honest_sets(), st.floats(-10, 10), st.floats(-10, 10))
@settings(max_examples=100, deadline=None)
def test_ipm_is_linear_in_eps(v, e1, e2):
    np.testing.assert_allclose(AT.craft(v, "ipm", e1 + e2), AT.craft(v, "ipm", e1) + AT.craft(v, "ipm", e2),
                               rtol=1e-9, atol=1e-9)


def test_alie_moves_z_population_stds_below_the_mean():
    v = np.array([[1.0, 5.0], [3.0, 5.0]])
    np.testing.assert_array_equal(AT.craft(v, "alie", 1.5), [2.0 - 1.5, 5.0])     # sigma = (1, 0), not (sqrt 2, 0)


def test_gauss_draw_depends_on_every_counter_word_and_the_key():
    base = AT.gauss_xi(64, 9, 4, 1, 50, 2)
    np.testing.assert_array_equal(base, AT.gauss_xi(64, 9, 4, 1, 50, 2))
    for other in (AT.gauss_xi(64, 9, 4, 2, 50, 2), AT.gauss_xi(64, 9, 4, 1, 50, 3), AT.gauss_xi(64, 9, 3, 1, 50, 2),
                  AT.gauss_xi(64, 9, 4, 1, 100, 2), AT.gauss_xi(64, 10, 4, 1, 50, 2), AT.gauss_xi(64, 9 << 32, 4, 1, 50, 2)):
        assert not np.any(other == base)
    np.testing.assert_allclose(AT.gauss_xi(64, 9, 4, 1, 50, 2, np.float32), base, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ oracle round / hook
def _team5(labels, seed=3):
    from rcmarl import nets
    rs = np.random.RandomState(seed)
    w = [[nets.glorot_uniform(10, 5, rs), nets.glorot_uniform(10, 1, rs), nets.glorot_uniform(15, 1, rs)] for _ in range(5)]
    in_nodes = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
    ags = TU.oracle_agents(labels, w, [1] * 5, [0.01] * 5, 0.9)
    s, ns, a, r = TU.grid_rows(rs, 40, 5, 5)
    return ags, in_nodes, (s, ns, a, r)


def _params(ags):
    return [np.concatenate([np.ravel(x) for n in ag.get_parameters() for x in n]) for ag in ags]


def test_update_round_without_a_hook_is_the_oracles():
    labels = ["Cooperative", "Malicious", "Cooperative", "Greedy", "Faulty"]
    ags, in_nodes, rows = _team5(labels)
    mine = copy.deepcopy(ags)
    kw = dict(n_envs=1, n_epochs=2, n_actor_steps=40, common_reward=False)
    want = O.update_round(ags, labels, in_nodes, *rows, perm_source=O.make_perm_source(1), **kw)
    got = AT.update_round(mine, labels, in_nodes, *rows, perm_source=O.make_perm_source(1), **kw)
    for k in want:
        np.testing.assert_array_equal(got[k], want[k])
    for x, y in zip(_params(mine), _params(ags)):
        np.testing.assert_array_equal(x, y)


def test_hook_replaces_only_the_byzantine_entries_with_per_receiver_messages():
    labels = ["Cooperative"] * 4 + ["Byzantine"]
    ags, in_nodes, _ = _team5(labels)
    msgs = [ag.critic for ag in ags]
    tmsgs = [ag.TR for ag in ags]
    hook = AT.make_hook(labels, in_nodes, {4: ("ipm", 0.5)})
    per_c, per_t = hook(0, msgs, tmsgs)
    assert AT.byzantine_pairs(labels, in_nodes) == [(4, 1, [1, 2, 3]), (4, 2, [2, 3, 0]), (4, 3, [3, 0, 1])]
    for j in range(4):
        for pos, i in enumerate(in_nodes[j]):
            if i != 4:
                assert per_c[j][pos] is msgs[i] and per_t[j][pos] is tmsgs[i]
            else:
                honest = [k for k in in_nodes[j] if k != 4]
                want = -0.5 * np.mean([AT.pack(msgs[k], np.float64) for k in honest], 0)
                np.testing.assert_allclose(AT.pack(per_c[j][pos], np.float64), want, rtol=1e-12, atol=1e-15)
    # different honest sets give different messages
    assert not np.allclose(AT.pack(per_c[1][3], np.float64), AT.pack(per_c[2][2], np.float64))


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_attack_job_layout_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = ["dst", "msgs", "msg_stride", "n", "n_honest", "honest", "kind", "param", "seed", "attacker", "receiver",
              "round", "epoch"]
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'printf("%zu", sizeof(rcmarl_attack_job));'
                   + "".join(f'printf(" %zu", offsetof(rcmarl_attack_job, {f}));' for f in fields)
                   + 'printf(" %d %d %d\\n", RCMARL_ATTACK_ALIE, RCMARL_ATTACK_IPM, RCMARL_ATTACK_GAUSS); return 0;}')
    exe = tmp_path / "off"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == ctypes.sizeof(L.AttackJob) == 128
    assert got[1:-3] == [getattr(L.AttackJob, f).offset for f in fields]
    assert got[-3:] == [L.ATTACK_ALIE, L.ATTACK_IPM, L.ATTACK_GAUSS] == [0, 1, 2]
    assert ("rcmarl_attack", ctypes.c_int, [ctypes.POINTER(L.AttackJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS


def _job(**kw):
    from rcmarl import _lib as L
    j = L.AttackJob()
    j.dst, j.msgs, j.n, j.n_honest, j.kind, j.param = 4096, 8192, 10, 2, L.ATTACK_ALIE, 1.0
    j.honest[0], j.honest[1] = 0, 1
    for k, v in kw.items():
        if k == "honest":
            for i, x in enumerate(v):
                j.honest[i] = x
        else:
            setattr(j, k, v)
    return j


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-3), dict(n_honest=0), dict(n_honest=17),
    dict(honest=[0, -1]), dict(kind=3), dict(kind=-1), dict(param=float("nan")), dict(param=float("inf")),
    dict(param=float("-inf")), dict(kind=2, param=-0.5), dict(attacker=256), dict(receiver=300),
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    good = _job()
    for jobs in ([_job(**bad)], [good, _job(**bad)]):
        arr = (L.AttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_attack(arr, len(arr), None) == -1                   # RCMARL_ERR_ARG


def test_library_refuses_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_attack(None, 1, None) == -1
    arr = (L.AttackJob * 33)(*[_job() for _ in range(33)])
    assert lib.rcmarl_attack(arr, 0, None) == -1
    assert lib.rcmarl_attack(arr, 33, None) == -1


def test_attack_names_and_parameters():
    from rcmarl import _lib as L
    assert L.check_attack(("alie", 1)) == (0, 1.0) and L.check_attack(("ipm", -2.5)) == (1, -2.5)
    assert L.check_attack(("gauss", 0)) == (2, 0.0)
    for bad in [("median", 1), ("gauss", -1e-3), ("alie", float("nan")), ("ipm", float("inf")), ("alie",), "alie",
                None, ("alie", "x"), (2, 1.0)]:
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)


# ------------------------------------------------------------------------------------------------ Trainer refusals
@pytest.fixture
def no_device(monkeypatch):
    """Trainer construction that reaches the device fails with DeviceTouched instead."""
    import torch
    from rcmarl import _lib

    _lib.lib()

    class DeviceTouched(Exception):
        pass

    def touched(*a, **k):
        raise DeviceTouched()
    monkeypatch.setattr(torch.cuda, "current_device", touched)
    return DeviceTouched


C5 = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]


def trainer(attack, labels=None, in_nodes=None, aggregation="clip", H=1):
    from rcmarl.trainer import Trainer
    labels = labels or ["Cooperative"] * 4 + ["Byzantine"]
    return Trainer(labels=labels, in_nodes=in_nodes or C5, weights=[], desired=np.zeros((len(labels), 2)), H=H,
                   aggregation=aggregation, attack=attack)


@pytest.mark.parametrize("attack,labels,in_nodes", [
    (None, None, None),                                                        # a Byzantine agent without an attack
    ([None] * 5, None, None),
    ([("alie", 1.0)] + [None] * 4, ["Cooperative"] * 4 + ["Faulty"], None),     # an attack on a non-Byzantine agent
    ([None] * 4 + [("ipm", 1.0)], ["Cooperative"] * 4 + ["Malicious"], None),
    ([None] * 3 + [("alie", 1.0)] * 2, None, None),                            # ... on a cooperative one
    (("median", 1.0), None, None),                                             # unknown name
    (("gauss", -0.1), None, None),                                             # bad parameters
    (("alie", float("nan")), None, None),
    (("ipm", float("inf")), None, None),
    ([None] * 4, None, None),                                                  # not one entry per agent
    (("alie", 1.0), ["Cooperative", "Malicious", "Greedy", "Cooperative", "Byzantine"],
     [[1, 2, 4], [1, 4], [2, 4, 1], [3, 4], [4, 0]]),                          # receiver 0 hears no cooperative agent
])
def test_trainer_refuses_invalid_attacks_before_any_device_work(no_device, attack, labels, in_nodes):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(attack, labels, in_nodes, H=0)


@pytest.mark.parametrize("attack,labels", [
    (("alie", 1.0), None),
    ([None] * 4 + [("gauss", 0.0)], None),
    (None, ["Cooperative"] * 4 + ["Faulty"]),
    (("ipm", 2.0), ["Cooperative"] * 4 + ["Faulty"]),                          # one pair for every Byzantine agent: none
    (("alie", 1.0), ["Byzantine"] * 5),                                        # no cooperative receiver, no pair
])
def test_trainer_accepts_valid_attacks(no_device, attack, labels):
    with pytest.raises(no_device):
        trainer(attack, labels)
