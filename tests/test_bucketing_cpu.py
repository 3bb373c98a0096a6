"""CPU checks of randomized bucketing (rcmarl_bucket_mix, include/rcmarl.h): the oracle's permutation, buckets, rows and
mixing matrix (tests/bucket_oracle.py) and each consequence the header states, a hand-worked example, the enum, struct
and symbol as gcc sees the header and the bindings declare them, the library's refusals without a device,
check_mixing's names and limits, the Trainer's refusals and message-row layout before it touches a device, and
build_trainer forwarding each agent's mixing."""
import ctypes
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import bucket_oracle as BO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@st.composite
def job(draw):
    """(n_in, s, (seed, receiver, net, round, epoch))."""
    n_in = draw(st.integers(1, 16))
    s = draw(st.integers(1, 17))
    words = (draw(st.integers(0, 2 ** 64 - 1)), draw(st.integers(0, 255)), draw(st.integers(0, 1)),
             draw(st.integers(0, 2 ** 32 - 1)), draw(st.integers(0, 2 ** 32 - 1)))
    return n_in, s, words


@given(job())
@settings(max_examples=300, deadline=None)
def test_pi_is_a_permutation_and_the_buckets_partition_the_received_slots(c):
    n_in, s, words = c
    pi = BO.permutation(n_in, *words)
    assert sorted(pi) == list(range(1, n_in))
    bks = BO.buckets(n_in, s, *words)
    assert len(bks) == BO.n_out(n_in, s) - 1 == -(-(n_in - 1) // s)
    assert sorted(l for b in bks for l in b) == list(range(1, n_in))
    assert all(len(b) == s for b in bks[:-1]) and all(1 <= len(b) <= s for b in bks)
    assert [sorted(pi[b:b + s]) for b in range(0, n_in - 1, s)] == bks


def test_each_slot_lands_in_each_position_about_equally_often():
    """Over 4000 counters (rounds), slot l sits at position q of pi about 4000 / m times: a loose chi^2 bound per
    n_in (the statistic has (m - 1)^2 degrees of freedom; 3x that is far out in its tail)."""
    for n_in in (3, 4, 8, 16):
        m = n_in - 1
        counts = np.zeros((m, m))
        trials = 4000
        for r in range(trials):
            pi = BO.permutation(n_in, 0x1234_5678_9ABC_DEF0, 3, r & 1, r, 11)
            for q, l in enumerate(pi):
                counts[l - 1, q] += 1
        want = trials / m
        chi2 = float(((counts - want) ** 2 / want).sum())
        assert chi2 < 3 * max((m - 1) ** 2, 1) + 10, (n_in, chi2)


def test_draws_depend_on_every_counter_word_and_the_seed():
    base = (99, 5, 0, 17, 2)
    pis = {tuple(BO.permutation(16, *base))}
    for k, v in enumerate((100, 6, 1, 18, 3)):
        w = list(base)
        w[k] = v
        pis.add(tuple(BO.permutation(16, *w)))
    assert len(pis) == 6
    assert BO.permutation(16, *base) == BO.permutation(16, *base)


def test_s1_gives_permuted_bitwise_copies_and_large_s_one_bucket():
    rs = np.random.RandomState(3)
    X = (rs.randn(9, 13) * 5).astype(np.float32)
    words = (42, 1, 0, 7, 0)
    Y, M = BO.bucket_mix(X, 1, *words)
    pi = BO.permutation(9, *words)
    np.testing.assert_array_equal(Y, X[[0] + pi])
    np.testing.assert_array_equal(M, np.eye(9, dtype=np.float32)[[0] + pi])
    for s in (8, 9, 1000, 2 ** 31 - 1):
        Y, M = BO.bucket_mix(X, s, *words)
        assert Y.shape == (2, 13)
        np.testing.assert_array_equal(Y[0], X[0])
        s32 = np.zeros(13, np.float32)
        for l in range(1, 9):
            s32 = s32 + X[l]
        np.testing.assert_array_equal(Y[1], s32 / np.float32(8))
        np.testing.assert_array_equal(M[1], [0] + [np.float32(1) / np.float32(8)] * 8)
    Y, M = BO.bucket_mix(X[:1], 2, *words)                      # n_in = 1: the own row only
    np.testing.assert_array_equal(Y, X[:1])
    np.testing.assert_array_equal(M, [[1]])


@given(job(), st.integers(0, 2 ** 31 - 1))
@settings(max_examples=200, deadline=None)
def test_rows_of_M_sum_to_one_and_M_reproduces_the_rows(c, seed):
    n_in, s, words = c
    rs = np.random.RandomState(seed)
    X = rs.randn(n_in, 7) * rs.uniform(0.1, 3, size=(n_in, 1))
    Y, M = BO.bucket_mix(X, s, *words)
    np.testing.assert_allclose(M.sum(1), 1.0, rtol=1e-15)
    assert M[0, 0] == 1 and (M[0, 1:] == 0).all() and (M[1:, 0] == 0).all()
    assert ((M[1:] > 0).sum(0)[1:] == 1).all()                   # each received slot in exactly one bucket
    np.testing.assert_allclose(Y, M @ X, rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(Y[0], X[0])


@pytest.mark.parametrize("poison", [np.inf, -np.inf, 1e30, "pm"])
def test_H_poisoned_inputs_give_at_most_H_poisoned_rows(poison):
    rs = np.random.RandomState(8)
    for n_in, s, H in ((4, 2, 1), (8, 2, 2), (16, 3, 3), (9, 4, 2), (16, 1, 5)):
        for r in range(20):
            X = rs.randn(n_in, 11).astype(np.float32)
            bad = rs.choice(np.arange(1, n_in), size=H, replace=False)
            for q, b in enumerate(bad):
                if poison == "pm":                               # +inf and -inf in one bucket give +inf, not NaN
                    X[b] = np.inf if q % 2 == 0 else -np.inf
                else:
                    X[b, ::2] = poison
            words = (r, 4, r & 1, 3 * r, 1)
            Y, M = BO.bucket_mix(X, s, *words)
            poisoned = [k for k in range(1, Y.shape[0]) if not np.isfinite(Y[k]).all()]
            assert len(poisoned) <= H
            for k in poisoned:
                assert (Y[k] == np.inf).all()
                assert set(np.flatnonzero(M[k])) & set(bad)
            for k in range(1, Y.shape[0]):
                if not set(np.flatnonzero(M[k])) & set(bad):
                    assert np.isfinite(Y[k]).all()


def test_hand_worked_example():
    """seed 7, receiver 2, net 1, round 5, epoch 3, n_in = 5 (m = 4): counter (0, 2 | 1 << 8 | 0x20000000, 5, 3) gives
    the words x = 0xa301eb19, y = 0x2be4ad92, z = 0xdd6b09da.  Fisher-Yates from pi = [1, 2, 3, 4]:
      i = 3: j = (x * 4) >> 32 = 2, swap pi[3], pi[2] -> [1, 2, 4, 3]
      i = 2: j = (y * 3) >> 32 = 0, swap pi[2], pi[0] -> [4, 2, 1, 3]
      i = 1: j = (z * 2) >> 32 = 1, no change.
    At s = 2 the buckets are {4, 2} and {1, 3}, summed as slot 2 + slot 4 and slot 1 + slot 3."""
    words = (7, 2, 1, 5, 3)
    assert BO.draws(3, *words) == [0xa301eb19, 0x2be4ad92, 0xdd6b09da]
    assert BO.permutation(5, *words) == [4, 2, 1, 3]
    assert BO.buckets(5, 2, *words) == [[2, 4], [1, 3]]
    assert BO.buckets(5, 3, *words) == [[1, 2, 4], [3]]
    X = np.array([[10.0, -1.0], [1.0, 2.0], [3.0, 4.0], [5.0, 6.0], [7.0, 8.0]], np.float32)
    Y, M = BO.bucket_mix(X, 2, *words)
    np.testing.assert_array_equal(Y, [[10.0, -1.0], [5.0, 6.0], [3.0, 4.0]])
    np.testing.assert_array_equal(M, [[1, 0, 0, 0, 0], [0, 0, 0.5, 0, 0.5], [0, 0.5, 0, 0.5, 0]])
    Y, M = BO.bucket_mix(X, 3, *words)
    np.testing.assert_array_equal(Y[1], (X[1] + X[2] + X[4]) / np.float32(3))
    np.testing.assert_array_equal(Y[2], X[3])


def test_oracle_refuses_what_the_library_refuses():
    for n_in, s in ((0, 2), (4, 0), (4, -1)):
        with pytest.raises(ValueError):
            BO.n_out(n_in, s)


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enum_struct_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = [f[0] for f in L.BucketJob._fields_]
    assert fields == ["dst", "msgs", "msg_stride", "weights_out", "n", "n_in", "s", "in_nodes", "seed", "receiver",
                      "net", "round", "epoch"]
    offs = " ".join(f'printf("%d ", (int)offsetof(rcmarl_bucket_job, {f}));' for f in fields)
    src = tmp_path / "bucket.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_bucket_job*, int, void*) = rcmarl_bucket_mix; (void)f;'
                   'rcmarl_mixing_rule a = RCMARL_MIX_NNM, b = RCMARL_MIX_BUCKET;'
                   f'printf("%d %d %d ", (int)a, (int)b, (int)sizeof(rcmarl_bucket_job)); {offs} return 0;}}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_bucket_mix(const rcmarl_bucket_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "bucket"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[:2] == [L.MIX_NNM, L.MIX_BUCKET] == [0, 1]
    assert got[2] == ctypes.sizeof(L.BucketJob)
    assert got[3:] == [getattr(L.BucketJob, f).offset for f in fields]
    assert ("rcmarl_bucket_mix", ctypes.c_int, [ctypes.POINTER(L.BucketJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_bucket_mix.argtypes == [ctypes.POINTER(L.BucketJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 rows of 100 floats, 1000 floats apart, its 3 dst rows (s = 2) far away at
    the same stride."""
    from rcmarl import _lib as L
    j = L.BucketJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.s = 1 << 24, 1 << 16, 1000, 100, 4, 2
    j.seed, j.receiver, j.net, j.round, j.epoch = 5, 3, 1, 9, 2
    for k in range(4):
        j.in_nodes[k] = k
    for k, v in kw.items():
        if k == "in_nodes":
            for i, x in enumerate(v):
                j.in_nodes[i] = x
        else:
            setattr(j, k, v)
    return j


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-5), dict(n_in=0), dict(n_in=17), dict(in_nodes=[0, 1, -1, 3]),
    dict(s=0), dict(s=-2), dict(net=2), dict(net=0xFFFFFFFF), dict(receiver=256), dict(receiver=1 << 20),
    dict(dst=(1 << 16) + 4 * 2000),                                           # dst row 0 on in-node row 2
    dict(dst=(1 << 16) - 4 * 2000),                                           # dst row 2 on in-node row 0
    dict(dst=(1 << 16) - 4 * 1000 + 4 * 99),                                  # dst row 0 ends inside in-node row 0
    dict(msg_stride=50),                                                      # dst rows overlap each other
    dict(weights_out=(1 << 16) + 4 * 1000 + 8), dict(weights_out=(1 << 16) - 4 * 3),   # weights_out on an in-node row
    dict(weights_out=(1 << 24) + 4 * 2050),                                   # ... on the job's dst row 2
    dict(weights_out=(1 << 24) - 4 * 11),                                     # 12 floats reaching dst row 0
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    for jobs in ([_job(**bad)], [_job(dst=1 << 26, weights_out=(1 << 26) + 4 * 8000), _job(**bad)]):
        arr = (L.BucketJob * len(jobs))(*jobs)
        assert lib.rcmarl_bucket_mix(arr, len(arr), None) == -1                   # RCMARL_ERR_ARG


def test_library_refuses_writes_on_another_jobs_ranges_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    arr = (L.BucketJob * 2)(_job(msgs=1 << 28), _job(dst=(1 << 28) - 4 * 1000))  # job 1's dst row 2 on job 0's row 1
    assert lib.rcmarl_bucket_mix(arr, 2, None) == -1
    first = dict(dst=1 << 26, weights_out=(1 << 26) + 4 * 8000)
    for second in (dict(dst=(1 << 26) + 4 * 99), dict(dst=(1 << 26) + 4 * 8000 - 4 * 2000),   # dst rows on first's
                   dict(weights_out=(1 << 26) + 4 * 2050), dict(weights_out=(1 << 26) + 4 * 8000 + 4 * 11)):
        arr = (L.BucketJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_bucket_mix(arr, 2, None) == -1, second
    assert lib.rcmarl_bucket_mix(None, 1, None) == -1
    arr = (L.BucketJob * 33)(*[_job(dst=(1 << 24) + 4 * 4000 * i) for i in range(33)])
    assert lib.rcmarl_bucket_mix(arr, 0, None) == -1
    assert lib.rcmarl_bucket_mix(arr, 33, None) == -1


def test_mixing_names_and_limits():
    from rcmarl import _lib as L
    for name in ("bucket", ("bucket", 1), ("bucket", 2), ("bucket", 15), ("bucket", np.int64(3)), ("bucket", 2 ** 31 - 1)):
        for H, n in ((0, 1), (1, 2), (15, 16), (0, 16), (3, 4)):
            assert L.check_mixing(name, H, n) == L.MIX_BUCKET == 1
    for H, n in ((1, 1), (-1, 4), (4, 4), (0, 0), (0, 17)):
        with pytest.raises(L.RcmarlError):
            L.check_mixing("bucket", H, n)
    for name in ("NNM", "bucketing", 0, "clip", None, ("bucket", 0), ("bucket", -1), ("bucket", 2.0), ("bucket", True),
                 ("bucket", 2 ** 31), ("bucket",), ("bucket", 2, 3), ["bucket", 2], ("nnm", 2), "Bucket"):
        with pytest.raises(L.RcmarlError):
            L.check_mixing(name, 0, 4)
    assert L.check_mixing("nnm", 1, 4) == L.MIX_NNM == 0
    assert L.MIXING_RULES == {"nnm": 0}
    assert L.mixing_entry(None) is None and L.mixing_entry("nnm") == "nnm"
    assert L.mixing_entry("bucket") == ("bucket", 2) == L.mixing_entry(("bucket", np.int32(2)))
    for n_in in range(1, 17):
        assert L.mixed_rows(None, n_in) == L.mixed_rows("nnm", n_in) == n_in
        for s in (1, 2, 3, 5, 16, 100):
            assert L.mixed_rows(("bucket", s), n_in) == BO.n_out(n_in, s)
        assert L.mixed_rows("bucket", n_in) == BO.n_out(n_in, 2)
    assert [L.mixed_rows("bucket", n) for n in (4, 8, 16)] == [3, 5, 9]


# ------------------------------------------------------------------------------------------------ Trainer
class DeviceTouched(Exception):
    pass


@pytest.fixture
def no_device(monkeypatch):
    """Trainer construction that reaches the device fails with DeviceTouched instead."""
    import torch
    from rcmarl import _lib

    _lib.lib()

    def touched(*a, **k):
        raise DeviceTouched()
    monkeypatch.setattr(torch.cuda, "current_device", touched)
    return DeviceTouched


C5 = [[0, 1, 2, 3], [1, 2, 3, 4], [2, 3, 4, 0], [3, 4, 0, 1], [4, 0, 1, 2]]
BYZ = ["Cooperative"] * 4 + ["Byzantine"]
MAL = ["Cooperative"] * 4 + ["Malicious"]


def trainer(mixing, aggregation="clip", H=1, labels=None, attack=None):
    from rcmarl.trainer import Trainer
    return Trainer(labels=labels or MAL, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing)


def built(excinfo):
    """The Trainer whose construction stopped at the device (from the frame of its __init__)."""
    tb = excinfo.tb
    while tb is not None:
        if tb.tb_frame.f_code.co_name == "__init__" and "mixing" in tb.tb_frame.f_locals:
            return tb.tb_frame.f_locals["self"]
        tb = tb.tb_next
    raise AssertionError("no Trainer frame")


@pytest.mark.parametrize("mixing,aggregation,H,labels,attack,match", [
    ("bucket", "krum", 1, None, None, "buckets its 4 messages into 3 rows"),       # krum needs n >= H + 3 = 4
    ("bucket", "mkrum", 1, BYZ, ("alie", 1.5), "buckets its 4 messages into 3 rows"),
    ([None, ("bucket", 2), None, None, None], ["clip", "mkrum", "clip", "clip", "clip"], 1, None, None, "agent 1"),
    (("bucket", 3), "trim", 1, None, None, "2H < n_in"),                            # 2 rows: trim needs 2H < 2
    (("bucket", 0), "clip", 1, None, None, "bucket size"),
    (("bucket", 2.0), "clip", 1, None, None, "bucket size"),
    ([None, None, ("bucket", -3), None, None], "clip", 1, None, None, "bucket size"),
    ([None, None, None, None, ("bucket", 0)], "clip", 1, None, None, "bucket size"),  # checked at any agent
    ("bucket", "clip", 1, BYZ, ("tailored_std", 2.0), "tailored attack does not model"),
    ([None, ("bucket", 2), None, None, None], "wmsr", 1, BYZ, ("tailored_uv", 1.0), "tailored attack does not model"),
])
def test_trainer_refuses_before_any_device_work(no_device, mixing, aggregation, H, labels, attack, match):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match=match):
        trainer(mixing, aggregation, H, labels, attack)


@pytest.mark.parametrize("mixing,aggregation,H,labels,attack", [
    ("bucket", "clip", 1, None, None), (("bucket", 1), "krum", 1, None, None), (("bucket", 5), "clip", 0, None, None),
    ("bucket", ["dnc", "trim", "gmed", "wmsr", "clip"], [1, 1, 1, 1, 0], BYZ, ("mimic", 5)),
    ("bucket", ["scclip", "clip", "trim", "wmsr", "clip"], 1, BYZ, ("alie", 1.5)),
    (["nnm", ("bucket", 2), None, "bucket", None], ["krum", "clip", "mkrum", "dnc", "clip"], 1, BYZ, ("gauss", 0.3)),
    ([("bucket", 2), None, None, None, None], "clip", 1, BYZ, ("tailored_std", 2.0)),   # agent 0 does not hear agent 4
])
def test_trainer_accepts_bucketing_alone_and_mixed(no_device, mixing, aggregation, H, labels, attack):
    with pytest.raises(no_device):
        trainer(mixing, aggregation, H, labels, attack)


def test_trainer_row_layout(no_device):
    """The mixed rows of nnm and bucketing agents follow the Byzantine pair, distance-based and dnc rows in mix_agents
    order: n_in rows for an nnm agent, n_out = 3 for a bucketing agent at n_in = 4 and s = 2 (2 at s = 3)."""
    with pytest.raises(no_device) as ex:
        trainer(["bucket", "nnm", None, ("bucket", 3), "bucket"], ["scclip", "dnc", "clip", "trim", "clip"],
                [1, 1, 1, 0, 0], BYZ, ("gauss", 0.3))
    tr = built(ex)
    assert [p[:2] for p in tr.byz_pairs] == [(4, 1), (4, 2), (4, 3)]
    assert tr.vec_row == {0: 8} and tr.dnc_row == {1: 9}
    assert tr.mixing == [("bucket", 2), "nnm", None, ("bucket", 3), None]
    assert tr.mix_agents == [0, 1, 3] and tr.mix_row == {0: 10, 1: 13, 3: 17}
    assert tr._rule_nodes(0) == [10, 11, 12] and tr._rule_nodes(1) == [13, 14, 15, 16]
    assert tr._rule_nodes(3) == [17, 18]
    assert tr._rule_nodes(2) == tr._receiver_nodes(2) == [2, 3, 6, 0]
    with pytest.raises(no_device) as ex:
        trainer(("bucket", 2), "clip", 1, BYZ, ("alie", 1.0))
    tr = built(ex)
    assert tr.mixing == [("bucket", 2)] * 4 + [None] and tr.mix_row == {0: 8, 1: 11, 2: 14, 3: 17}


def test_build_trainer_forwards_each_agents_mixing(no_device):
    """train_RPBCAC builds its Trainer with mixing=[agent.mixing], so an agent's nnm or bucketing is honoured."""
    from training.train_agents import build_trainer

    def agent(mixing, H=1):
        return types.SimpleNamespace(get_parameters=lambda: [], H=H, aggregation="clip", mixing=mixing)
    env = types.SimpleNamespace(std_state=1, mean_state=0, randomize_state=True, desired_state=np.zeros((5, 2)),
                                n_envs=4, nrow=5, ncol=5)
    args = dict(agent_label=MAL, in_nodes=C5, gamma=0.9, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=100,
                common_reward=False, random_seed=3)
    agents = [agent(("bucket", 2)), agent("nnm"), agent(None), agent(("bucket", 3)),
              types.SimpleNamespace(get_parameters=lambda: [], H=0)]        # an adversary has no mixing attribute
    with pytest.raises(no_device) as ex:
        build_trainer(env, agents, args)
    tr = built(ex)
    assert tr.mixing == [("bucket", 2), "nnm", None, ("bucket", 3), None] and tr.mix_agents == [0, 1, 3]
    with pytest.raises(no_device) as ex:
        build_trainer(env, [agent(None) for _ in range(4)] + [agents[-1]], args)
    assert built(ex).mix_agents == []
