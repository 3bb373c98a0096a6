"""CPU checks of adaptive robust clipping (rcmarl_arc_clip, include/rcmarl.h): the k_clip table, the oracle's properties
(tests/arc_oracle.py) -- H = 0 is the identity, row 0 never changes, at most k_clip rows change, every clipped row lies
at distance tau from x_0, non-finite slots become x_0 -- a hand-worked example, the enum and symbol as gcc sees the
header and the bindings declare them, the library's refusals without a device, check_clipping and arc_count, and the
Trainer's, build_trainer's and RPBCAC_agent's refusals and row layout before any device work."""
import ctypes
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import arc_oracle as AO
from test_bucketing_cpu import C5, BYZ, MAL, DeviceTouched, no_device   # noqa: F401  (no_device is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32, f64 = np.float32, np.float64


def _data(seed, n, P, dtype=f64):
    rs = np.random.RandomState(seed)
    X = rs.randn(P) + rs.randn(n, P) * rs.uniform(0.05, 3.0, size=(n, 1))
    return X.astype(dtype)


# ------------------------------------------------------------------------------------------------ oracle
def test_k_clip_table():
    """k_clip = (2 H (n - H)) // n over n = 1 .. 16, H = 0 .. n - 1; the library's arc_count agrees."""
    from rcmarl import _lib as L
    want = {1: [0], 2: [0, 1], 3: [0, 1, 1], 4: [0, 1, 2, 1], 5: [0, 1, 2, 2, 1], 16: [0, 1, 3, 4, 6, 6, 7, 7, 8, 7,
                                                                                       7, 6, 6, 4, 3, 1]}
    for n in range(1, 17):
        row = [AO.k_clip(H, n) for H in range(n)]
        assert row == [L.arc_count(H, n) for H in range(n)]
        assert row == [int(np.floor(2 * (H / n) * (n - H) + 1e-9)) for H in range(n)]
        assert row[0] == 0 and max(row) <= n // 2
        if n in want:
            assert row == want[n], n
    assert AO.k_clip(1, 4) == 1                                 # the C2 shape
    assert [(n, H) for n in range(2, 17) for H in range(n) if AO.k_clip(H, n) >= n - 1] == [(2, 1)]   # tau = 0


@given(st.integers(1, 16), st.integers(1, 200), st.integers(0, 2 ** 31 - 1))
@settings(max_examples=100, deadline=None)
def test_h0_is_the_identity_and_row_0_never_changes(n, P, seed):
    rs = np.random.RandomState(seed)
    for dtype in (f32, f64):
        X = _data(seed, n, P, dtype)
        Y, c, _ = AO.clip(X, 0)
        np.testing.assert_array_equal(Y, X)
        assert (c == 1).all()
        H = int(rs.randint(0, n))
        Y, c, _ = AO.clip(X, H)
        np.testing.assert_array_equal(Y[0], X[0])
        assert c[0] == 1


@given(st.integers(2, 16), st.integers(1, 200), st.integers(0, 2 ** 31 - 1))
@settings(max_examples=150, deadline=None)
def test_at_most_k_clip_rows_change_and_each_lies_at_distance_tau(n, P, seed):
    rs = np.random.RandomState(seed)
    H = int(rs.randint(0, n))
    X = _data(seed, n, P)
    Y, c, tau = AO.clip(X, H)
    changed = [k for k in range(n) if not np.array_equal(Y[k], X[k])]
    assert len(changed) <= AO.k_clip(H, n)
    d_in, d_out = AO.distances(X), AO.distances(Y)
    for k in changed:
        assert d_in[k] > tau
        np.testing.assert_allclose(d_out[k], tau, rtol=1e-12, atol=1e-12 * d_in[k])
    assert (d_out <= max(tau, 0) * (1 + 1e-12) + 1e-300).all() or AO.k_clip(H, n) == 0
    # the clipped rows lie on the segment from x_0 to x_k
    for k in changed:
        np.testing.assert_allclose(Y[k], X[0] + c[k] * (X[k] - X[0]), rtol=0, atol=1e-12 * np.abs(X).max())
    # fp32: each changed row is x_0 + c (x_k - x_0) rounded per operation, within a few ulps of distance tau
    X32 = X.astype(f32)
    c32, tau32 = AO.factors(X32, H)
    Y32 = AO.rows(X32, c32)
    for k in range(1, n):
        if c32[k] not in (0.0, 1.0):
            np.testing.assert_allclose(np.linalg.norm(Y32[k].astype(f64) - X32[0]), tau32, rtol=1e-5)


@pytest.mark.parametrize("poison", [np.inf, -np.inf, 1e30])
def test_non_finite_slots_become_x0(poison):
    X = _data(7, 6, 50, f32)
    X[2, 3] = poison
    X[4] = poison
    for H in range(6):
        Y, c, _ = AO.clip(X, H)
        assert c[2] == c[4] == 0
        np.testing.assert_array_equal(Y[2], X[0])
        np.testing.assert_array_equal(Y[4], X[0])
        assert np.isfinite(Y).all()


def test_hand_worked_example():
    """n = 4, H = 1: k_clip = 1, so the furthest slot is pulled in to the second-furthest distance."""
    X = np.array([[0.0, 0.0], [3.0, 4.0], [0.0, 1.0], [6.0, 8.0]], f32)        # d = 5, 1, 10
    Y, c, tau = AO.clip(X, 1)
    assert tau == 5.0
    np.testing.assert_array_equal(c, [1.0, 1.0, 1.0, 0.5])
    np.testing.assert_array_equal(Y, [[0, 0], [3, 4], [0, 1], [3, 4]])
    Y, c, tau = AO.clip(X, 2)                                                # k_clip = 2: tau = 1
    assert tau == 1.0
    np.testing.assert_array_equal(c, [1.0, 0.2, 1.0, 0.1])
    np.testing.assert_array_equal(Y[3], (X[0] + f32(0.1) * (X[3] - X[0])).astype(f32))
    # ties: equal distances are either all kept or all clipped, only the value of tau matters
    X = np.array([[1.0], [2.0], [0.0], [3.0], [-1.0]], f32)                  # d = 1, 1, 2, 2
    Y, c, tau = AO.clip(X, 1)                                                # n = 5, H = 1: k_clip = 1, tau = 2
    assert tau == 2.0 and (c == 1).all()
    Y, c, tau = AO.clip(np.array([[0.0], [5.0]], f32), 1)                    # n = 2, H = 1: tau = 0
    assert tau == 0 and c[1] == 0 and Y[1, 0] == 0


def test_the_hook_clips_only_receivers_that_clip():
    rs = np.random.RandomState(4)
    shapes = [(2, 3), (3,)]
    msgs = [[rs.randn(*s) * (10 if i == 2 else 1) for s in shapes] for i in range(3)]
    labels = ["Cooperative", "Cooperative", "Byzantine"]
    in_nodes = [[0, 1, 2], [1, 0, 2], [2]]
    log = {}
    hook = AO.ArcHook(labels, in_nodes, ["arc", None, None], [1, 1, 0], log=log)
    per_c, per_t = hook(0, msgs, msgs)
    assert per_c[1] == [msgs[1], msgs[0], msgs[2]]
    X, c, tau = log[0][0][0]
    Y = np.stack([AO.AT.pack(m, f64) for m in per_c[0]])
    np.testing.assert_array_equal(Y, AO.clip(X, 1)[0])
    assert c[2] < 1 and sorted(log) == [0]


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enum_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "arc.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_vector_job*, int, void*) = rcmarl_arc_clip; (void)f;'
                   'rcmarl_mixing_rule a = RCMARL_MIX_ARC;'
                   'printf("%d %d", (int)a, (int)RCMARL_MIX_MOMENTUM); return 0;}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_arc_clip(const rcmarl_vector_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "arc"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [L.MIX_ARC, L.MIX_MOMENTUM] == [3, 2]
    assert ("rcmarl_arc_clip", ctypes.c_int, [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_arc_clip.argtypes == [ctypes.POINTER(L.VectorJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 in-node rows of 100 floats, 1000 floats apart; its 4 dst rows far away at
    the same stride, and its 4 weights elsewhere."""
    from rcmarl import _lib as L
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = 1 << 24, 1 << 16, 1000, 100, 4, 1, L.MIX_ARC
    j.weights_out = 1 << 22
    for k in range(4):
        j.in_nodes[k] = k
    for k, v in kw.items():
        if k == "in_nodes":
            for i, x in enumerate(v):
                j.in_nodes[i] = x
        else:
            setattr(j, k, v)
    return j


BAD = [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-5), dict(n_in=0), dict(n_in=17), dict(in_nodes=[0, 1, -1, 3]),
    dict(rule=0), dict(rule=1), dict(rule=2), dict(rule=4), dict(H=-1), dict(H=4), dict(n_in=1, H=1),
    dict(dst=(1 << 16) + 4 * 2000),                                           # dst row 0 on in-node row 2
    dict(dst=(1 << 16) - 4 * 3000),                                           # dst row 3 on in-node row 0
    dict(dst=(1 << 16) - 4 * 1000 + 4 * 99),                                  # dst row 0 ends inside in-node row 0
    dict(msg_stride=50),                                                      # dst rows overlap each other
    dict(weights_out=(1 << 16) + 4 * 1098),                                   # weights end inside in-node row 1
    dict(weights_out=(1 << 24) + 4 * 2000 + 4 * 99),                          # weights on dst row 2
]


@pytest.mark.parametrize("bad", BAD)
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    other = dict(dst=1 << 26, weights_out=1 << 25)
    for jobs in ([_job(**bad)], [_job(**other), _job(**bad)]):
        arr = (L.VectorJob * len(jobs))(*jobs)
        assert lib.rcmarl_arc_clip(arr, len(arr), None) == -1                     # RCMARL_ERR_ARG


def test_library_refuses_ranges_of_another_job_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    first = dict(dst=1 << 26, weights_out=1 << 25)
    for second in (dict(dst=(1 << 26) + 4 * 3000 + 4 * 99),                  # dst rows on the first job's dst row 3
                   dict(weights_out=(1 << 26) + 4 * 10),                     # weights on its dst row 0
                   dict(weights_out=(1 << 25) + 4 * 3),                      # ... on its weights
                   dict(dst=(1 << 25) - 4 * 50),                             # dst row 0 on its weights
                   dict(msgs=(1 << 26) + 4 * 2000),                          # in-node rows on its dst rows
                   dict(msgs=(1 << 25) - 4 * 10)):                           # ... on its weights
        arr = (L.VectorJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_arc_clip(arr, 2, None) == -1, second
    assert lib.rcmarl_arc_clip(None, 1, None) == -1
    arr = (L.VectorJob * 33)(*[_job(dst=(1 << 24) + 4 * 4000 * i, weights_out=(1 << 22) + 64 * i) for i in range(33)])
    assert lib.rcmarl_arc_clip(arr, 0, None) == -1
    assert lib.rcmarl_arc_clip(arr, 33, None) == -1


def test_library_accepts_good_jobs_up_to_the_launch_without_a_device():
    """Valid tables pass every check and fail only at the launch (RCMARL_ERR_CUDA, no device here); the boundary: a
    dst row that starts where an in-node row ends is accepted, and P has no staging bound."""
    import sys
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_arc_cpu as T; from rcmarl import _lib as L; "
            "lib = L.lib(); "
            "jobs = [T._job(), T._job(dst=(1 << 26), weights_out=None, H=0), T._job(dst=(1 << 16) + 4 * 3100), "
            "        T._job(dst=1 << 28, n=10 ** 6, msg_stride=10 ** 6, msgs=1 << 30, weights_out=1 << 27)]; "
            "codes = [lib.rcmarl_arc_clip((L.VectorJob * 1)(j), 1, None) for j in jobs]; "
            "print(' '.join(map(str, codes)))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code, os.path.dirname(os.path.abspath(__file__)),
                          os.path.join(ROOT, "resilient-consensus-based-marl_b200")], capture_output=True, text=True,
                         env=env, timeout=120)
    assert out.returncode == 0, out.stderr
    assert [int(x) for x in out.stdout.split()] == [-3] * 4                        # RCMARL_ERR_CUDA


def test_check_clipping_accepts_exactly_none_and_arc():
    from rcmarl import _lib as L
    assert L.check_clipping(None) is None and L.check_clipping("arc") == "arc"
    for bad in ("ARC", "nnm", "clip", "", 3, True, ("arc",), ["arc"], "arc "):
        with pytest.raises(L.RcmarlError, match="clipping"):
            L.check_clipping(bad)


# ------------------------------------------------------------------------------------------------ Trainer
def trainer(clipping, mixing=None, aggregation="clip", H=1, labels=None, attack=None, momentum=None):
    from rcmarl.trainer import Trainer
    return Trainer(labels=labels or MAL, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing, momentum=momentum, clipping=clipping)


def built(excinfo):
    tb = excinfo.tb
    while tb is not None:
        if tb.tb_frame.f_code.co_name == "__init__" and "clipping" in tb.tb_frame.f_locals:
            return tb.tb_frame.f_locals["self"]
        tb = tb.tb_next
    raise AssertionError("no Trainer frame")


@pytest.mark.parametrize("clipping,mixing,aggregation,labels,attack,match", [
    ("ARC", None, "clip", None, None, "unknown clipping"),
    ("nnm", None, "clip", None, None, "unknown clipping"),
    ([None, None, None, None, "cc"], None, "clip", None, None, "unknown clipping"),     # checked at any agent
    (["arc", "arc"], None, "clip", None, None, "one entry per agent"),
    ("arc", None, "clip", BYZ, ("tailored_std", 2.0), "tailored attack against agent 1, whose clipping"),
    ([None, None, "arc", None, None], None, "scclip", BYZ, ("pipeline_uv", 1.0), "pipeline attack against agent 2"),
    ([None, None, None, "arc", None], None, "clip", BYZ, ("history_std", 2.0), "history attack against agent 3"),
    ("arc", ("bucket", 2), "krum", None, None, "buckets its 4 messages into 3 rows"),   # the rule check is unchanged
])
def test_trainer_refuses_before_any_device_work(no_device, clipping, mixing, aggregation, labels, attack, match):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match=match):
        trainer(clipping, mixing, aggregation, 1, labels, attack)


@pytest.mark.parametrize("clipping,mixing,momentum,aggregation,labels,attack", [
    ("arc", None, None, "clip", None, None), ("arc", "nnm", None, "krum", None, None),
    ("arc", ("bucket", 2), None, "dnc", None, None), ("arc", None, 0.9, "mda", BYZ, ("mimic", 5)),
    (["arc", None, "arc", None, None], [None, "nnm", ("bucket", 2), None, None], [None, None, None, 0.9, None],
     ["scclip", "clip", "trim", "smea", "clip"], BYZ, ("minsum_uv", 1.0)),
    ([None, None, None, None, "arc"], "nnm", None, "clip", None, None),              # a Malicious agent's entry is ignored
    (["arc", None, None, None, None], None, None, "clip", BYZ, ("tailored_std", 2.0)),  # agent 0 does not hear agent 4
    ("arc", None, None, "clip", BYZ, ("dissensus", 1.0)),
])
def test_trainer_accepts_clipping_alone_and_composed(no_device, clipping, mixing, momentum, aggregation, labels, attack):
    with pytest.raises(no_device):
        trainer(clipping, mixing, aggregation, 1, labels, attack, momentum)


def test_trainer_row_layout(no_device):
    """The clipped rows, n_in per agent in arc_agents order, follow the momentum rows; an agent's mixing step reads
    them, and so does its rule when it does not mix; a momentum agent's clipping reads its momentum rows."""
    with pytest.raises(no_device) as ex:
        trainer(["arc", "arc", None, "arc", "arc"], [None, "nnm", None, None, None], ["scclip", "clip", "dnc", "clip", "clip"],
                1, BYZ, ("gauss", 0.3), [None, None, None, 0.9, None])
    tr = built(ex)
    assert [p[:2] for p in tr.byz_pairs] == [(4, 1), (4, 2), (4, 3)]
    assert tr.vec_row == {0: 8} and tr.dnc_row == {2: 9} and tr.mix_row == {1: 10} and tr.mom_row == {3: 14}
    assert tr.clipping == ["arc", "arc", None, "arc", None] and tr.arc_agents == [0, 1, 3]
    assert tr.arc_row == {0: 18, 1: 22, 3: 26}
    assert tr._rule_nodes(0) == [18, 19, 20, 21] and tr._momentum_nodes(0) == [0, 1, 2, 3]
    assert tr._rule_nodes(1) == [10, 11, 12, 13] and tr._clipped_nodes(1) == [22, 23, 24, 25]
    assert tr._momentum_nodes(1) == [1, 2, 3, 5]
    assert tr._rule_nodes(3) == [26, 27, 28, 29] and tr._momentum_nodes(3) == [14, 15, 16, 17]
    assert tr._rule_nodes(2) == tr._receiver_nodes(2) == [2, 3, 6, 0]
    with pytest.raises(no_device) as ex:
        trainer(None, "nnm", "clip", 1, BYZ, ("alie", 1.0))
    tr = built(ex)
    assert tr.clipping == [None] * 5 and tr.arc_agents == [] and tr.arc_row == {}
    assert tr._clipped_nodes(1) == tr._receiver_nodes(1) and tr._rule_nodes(1) == [12, 13, 14, 15]


def test_build_trainer_forwards_each_agents_clipping(no_device):
    """train_RPBCAC builds its Trainer with clipping=[agent.clipping]; an adversary has no such attribute."""
    from training.train_agents import build_trainer

    def agent(clipping, H=1):
        return types.SimpleNamespace(get_parameters=lambda: [], H=H, aggregation="clip", mixing=None, momentum=None,
                                     clipping=clipping)
    env = types.SimpleNamespace(std_state=1, mean_state=0, randomize_state=True, desired_state=np.zeros((5, 2)),
                                n_envs=4, nrow=5, ncol=5)
    args = dict(agent_label=MAL, in_nodes=C5, gamma=0.9, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=100,
                common_reward=False, random_seed=3)
    agents = [agent("arc"), agent(None), agent("arc"), agent(None), types.SimpleNamespace(get_parameters=lambda: [], H=0)]
    with pytest.raises(no_device) as ex:
        build_trainer(env, agents, args)
    tr = built(ex)
    assert tr.clipping == ["arc", None, "arc", None, None] and tr.arc_agents == [0, 2]
    with pytest.raises(no_device) as ex:
        build_trainer(env, [agent(None) for _ in range(4)] + [agents[-1]], args)
    assert built(ex).arc_agents == []


def test_agent_refuses_bad_clipping_before_touching_its_models():
    """RPBCAC_agent checks the clipping name before it reads its models (stand-ins here)."""
    from rcmarl import _lib as L
    from agents.resilient_CAC_agents import RPBCAC_agent
    m = types.SimpleNamespace()
    for bad in ("ARC", "nnm", 1, ["arc"]):
        with pytest.raises(L.RcmarlError, match="clipping"):
            RPBCAC_agent(m, m, m, 0.002, 0.01, H=1, clipping=bad)
