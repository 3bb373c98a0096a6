"""CPU checks of per-neighbour momentum (rcmarl_momentum_mix, include/rcmarl.h): the oracle's properties
(tests/momentum_oracle.py) -- beta = 0 passes the messages through up to rounding, first ignores the old state,
poisoned coordinates stay poisoned, a common offset leaves M unchanged in fp64 -- the enum, struct and symbol as gcc
sees the header and the bindings declare them, the library's refusals without a device, check_momentum, and the
Trainer's, build_trainer's and RPBCAC_agent's refusals and row layout before any device work."""
import ctypes
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import momentum_oracle as MO
from test_bucketing_cpu import C5, BYZ, MAL, DeviceTouched, no_device   # noqa: F401  (no_device is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32, f64 = np.float32, np.float64


def _data(seed, n, P, dtype=f32):
    rs = np.random.RandomState(seed)
    c = rs.randn(P)
    X = c + rs.randn(n, P) * rs.uniform(0.05, 2.0, size=(n, 1))
    M = rs.randn(n, P) * 0.5
    return X.astype(dtype), c.astype(dtype), M.astype(dtype)


# ------------------------------------------------------------------------------------------------ oracle
@given(st.integers(1, 16), st.integers(1, 300), st.integers(0, 2 ** 31 - 1), st.booleans())
@settings(max_examples=100, deadline=None)
def test_beta_zero_gives_the_messages_up_to_one_rounding(n, P, seed, first):
    X, c, M = _data(seed, n, P)
    rows, new = MO.step(X, c, M, 0.0, first)
    np.testing.assert_array_equal(new, X - c)
    np.testing.assert_array_equal(rows, (X - c) + c)
    scale = np.maximum(np.abs(X), np.abs(c))
    assert (np.abs(rows - X) <= np.spacing(scale.astype(f32)) * 2).all()
    rows64, _ = MO.step(X.astype(f64), c.astype(f64), M.astype(f64), 0.0, first)
    np.testing.assert_allclose(rows64, X.astype(f64), rtol=0, atol=1e-12 * max(np.abs(X).max(), 1))


@pytest.mark.parametrize("dtype", [f32, f64])
def test_first_ignores_the_old_state(dtype):
    X, c, M = _data(1, 7, 50, dtype)
    want = MO.step(X, c, None, 0.9, True)
    for old in (M, np.full_like(M, np.inf), np.full_like(M, -np.inf), np.full_like(M, np.nan), M * 1e30):
        got = MO.step(X, c, old, 0.9, True)
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
        np.testing.assert_array_equal(got[1], X - c)


@pytest.mark.parametrize("beta", [0.0, 0.5, 0.9, 0.99])
def test_the_update_in_fp32_is_each_operation_rounded_on_its_own(beta):
    X, c, M = _data(2, 5, 333)
    rows, new = MO.step(X, c, M, beta, False)
    b = f32(beta)
    u = (X - c).astype(f32)
    want = (b * M).astype(f32) + ((f32(1) - b) * u).astype(f32)
    np.testing.assert_array_equal(new, want)
    np.testing.assert_array_equal(rows, (c + want).astype(f32))
    assert new.dtype == rows.dtype == f32


@pytest.mark.parametrize("dtype", [f32, f64])
def test_poisoned_coordinates_are_sticky_and_stay_in_their_slot(dtype):
    X, c, M = _data(3, 6, 40, dtype)
    M[2, ::3] = np.inf
    M[4, 1::5] = -np.inf
    rows, new = MO.step(X, c, M, 0.9, False)
    assert (new[2, ::3] == np.inf).all() and (new[4, 1::5] == -np.inf).all()
    assert (rows[2, ::3] == np.inf).all() and (rows[4, 1::5] == -np.inf).all()
    # a non-finite message coordinate replaces a finite M there, and stays
    X2 = X.copy()
    X2[1, :7] = np.inf
    X2[3, 5] = -np.inf
    rows2, new2 = MO.step(X2, c, new, 0.5, False)
    assert (new2[1, :7] == np.inf).all() and new2[3, 5] == -np.inf
    for _ in range(3):                                     # later finite messages do not heal it
        rows2, new2 = MO.step(X, c, new2, 0.5, False)
    assert (new2[1, :7] == np.inf).all() and new2[3, 5] == -np.inf and (new2[2, ::3] == np.inf).all()
    finite_slots = [0, 5]
    assert np.isfinite(rows2[finite_slots]).all()
    # a 1e30 message is finite: its slot's M grows, and only that row is far off
    X3 = X.copy()
    X3[5] = dtype(1e30)
    rows3, _ = MO.step(X3, c, MO.step(X, c, None, 0.9, True)[1], 0.9, False)
    assert (np.abs(rows3 - c).max(1) > 1e20).tolist() == [False] * 5 + [True]


@given(st.integers(1, 16), st.integers(1, 200), st.integers(0, 2 ** 31 - 1),
       st.sampled_from([0.0, 0.5, 0.9, 0.99]), st.integers(-8, 8))
@settings(max_examples=100, deadline=None)
def test_a_common_offset_leaves_M_unchanged_and_moves_every_row_in_fp64(n, P, seed, beta, e):
    """In fp64 a dyadic offset t (added exactly to inputs of at most 2^-10 .. 2^10) cancels in u = x - c: M is the same
    bit for bit over steps, and every row moves by t (up to the rounding of c + M)."""
    rs = np.random.RandomState(seed)
    t = 2.0 ** e * (1 + rs.randint(0, 8))
    c = np.round(rs.randn(P) * 64) / 64
    M = None
    Ms = None
    for k in range(3):
        X = c + np.round(rs.randn(n, P) * 1024) / 1024
        r0, M = MO.step(X, c, M, beta, k == 0)
        r1, Ms = MO.step(X + t, c + t, Ms, beta, k == 0)
        np.testing.assert_array_equal(M, Ms)
        np.testing.assert_allclose(r1, r0 + t, rtol=0, atol=1e-12 * (abs(t) + np.abs(r0).max() + 1))


def test_hand_worked_example():
    X = np.array([[3.0, 1.0], [5.0, -1.0]], f32)
    c = np.array([1.0, 1.0], f32)
    rows, M = MO.step(X, c, None, 0.5, True)
    np.testing.assert_array_equal(M, [[2.0, 0.0], [4.0, -2.0]])
    np.testing.assert_array_equal(rows, X)
    rows, M = MO.step(np.array([[1.0, 1.0], [1.0, 3.0]], f32), c, M, 0.5, False)
    np.testing.assert_array_equal(M, [[1.0, 0.0], [2.0, 0.0]])                 # 0.5 M + 0.5 u
    np.testing.assert_array_equal(rows, [[2.0, 1.0], [3.0, 1.0]])


def test_the_hook_carries_the_state_and_passes_other_receivers_through():
    class Ag:
        def __init__(self, c, t):
            self.c, self.t = c, t

        def get_parameters(self):
            return [None, self.c, self.t]
    rs = np.random.RandomState(4)
    shapes = [(2, 3), (3,)]
    msgs = [[rs.randn(*s) for s in shapes] for _ in range(3)]
    agents = [Ag([rs.randn(*s) for s in shapes], [rs.randn(*s) for s in shapes]) for _ in range(3)]
    labels = ["Cooperative", "Cooperative", "Byzantine"]
    in_nodes = [[0, 1, 2], [1, 0], [2]]
    log = {}
    hook = MO.MomentumHook(agents, labels, in_nodes, [0.9, None, None], log=log)
    for epoch in range(3):
        per_c, per_t = hook(epoch, msgs, msgs)
        assert per_c[1] == [msgs[1], msgs[0]] and len(per_c[0]) == 3
        X, c, rows, M = log[0][epoch][0]
        np.testing.assert_array_equal(X, np.stack([MO.AT.pack(msgs[k], f64) for k in in_nodes[0]]))
        np.testing.assert_array_equal(c, MO.AT.pack(agents[0].c, f64))
        if epoch == 0:
            np.testing.assert_array_equal(M, X - c)
        np.testing.assert_array_equal(MO.AT.pack(per_c[0][1], f64), rows[1])
    assert sorted(log) == [0] and len(log[0]) == 3


# ------------------------------------------------------------------------------------------------ C ABI / bindings
FIELDS = ["dst", "msgs", "msg_stride", "ref", "momentum", "momentum_stride", "n", "n_in", "in_nodes", "beta", "first"]


def test_enum_struct_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    assert [f[0] for f in L.MomentumJob._fields_] == FIELDS
    offs = " ".join(f'printf("%d ", (int)offsetof(rcmarl_momentum_job, {f}));' for f in FIELDS)
    src = tmp_path / "momentum.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_momentum_job*, int, void*) = rcmarl_momentum_mix; (void)f;'
                   'rcmarl_mixing_rule a = RCMARL_MIX_MOMENTUM;'
                   f'printf("%d %d ", (int)a, (int)sizeof(rcmarl_momentum_job)); {offs} return 0;}}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_momentum_mix(const rcmarl_momentum_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "momentum"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == L.MIX_MOMENTUM == 2
    assert got[1] == ctypes.sizeof(L.MomentumJob) == 128                     # 32 jobs fill 4 KB of kernel parameters
    assert got[2:] == [getattr(L.MomentumJob, f).offset for f in FIELDS]
    assert ("rcmarl_momentum_mix", ctypes.c_int, [ctypes.POINTER(L.MomentumJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.lib().rcmarl_momentum_mix.argtypes == [ctypes.POINTER(L.MomentumJob), ctypes.c_int, L.c_fp]


def _job(**kw):
    """A valid job on made-up addresses: 4 in-node rows of 100 floats, 1000 floats apart; its 4 dst rows far away at
    the same stride, its 4 M rows elsewhere 500 floats apart, and its ref elsewhere again."""
    from rcmarl import _lib as L
    j = L.MomentumJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_in = 1 << 24, 1 << 16, 1000, 100, 4
    j.ref, j.momentum, j.momentum_stride, j.beta, j.first = 1 << 22, 1 << 23, 500, 0.9, 0
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
    dict(dst=None), dict(msgs=None), dict(ref=None), dict(momentum=None), dict(n=0), dict(n=-5), dict(n_in=0),
    dict(n_in=17), dict(in_nodes=[0, 1, -1, 3]), dict(beta=1.0), dict(beta=1.5), dict(beta=-0.1), dict(beta=float("inf")),
    dict(beta=float("nan")), dict(beta=-float("inf")), dict(first=2), dict(first=-1),
    dict(dst=(1 << 16) + 4 * 2000),                                           # dst row 0 on in-node row 2
    dict(dst=(1 << 16) - 4 * 3000),                                           # dst row 3 on in-node row 0
    dict(dst=(1 << 16) - 4 * 1000 + 4 * 99),                                  # dst row 0 ends inside in-node row 0
    dict(msg_stride=50),                                                      # dst rows overlap each other
    dict(momentum=(1 << 16) + 4 * 1050),                                      # M row 0 on in-node row 1
    dict(momentum_stride=99),                                                 # M rows overlap each other
    dict(momentum=(1 << 24) + 4 * 2000 - 4 * 500),                            # M row 1 on dst row 2
    dict(ref=(1 << 16) + 4 * 3000 + 4 * 99),                                  # ref on in-node row 3
    dict(ref=(1 << 24) + 4 * 1000 + 4 * 50),                                  # ref on dst row 1
    dict(ref=(1 << 23) + 4 * 1500),                                           # ref on M row 3
]


@pytest.mark.parametrize("bad", BAD)
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    other = dict(dst=1 << 26, momentum=1 << 27, ref=1 << 25)
    for jobs in ([_job(**bad)], [_job(**other), _job(**bad)]):
        arr = (L.MomentumJob * len(jobs))(*jobs)
        assert lib.rcmarl_momentum_mix(arr, len(arr), None) == -1                 # RCMARL_ERR_ARG


def test_library_refuses_ranges_of_another_job_and_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    first = dict(dst=1 << 26, momentum=1 << 27, ref=1 << 25)
    for second in (dict(dst=(1 << 26) + 4 * 3000 + 4 * 99),                  # dst rows on the first job's dst row 3
                   dict(momentum=(1 << 26) + 4 * 10),                        # M rows on its dst rows
                   dict(momentum=(1 << 27) + 4 * 1499),                      # ... on its M row 3
                   dict(dst=(1 << 25) - 4 * 50),                             # dst row 0 on its ref
                   dict(momentum=(1 << 25) - 4 * 1550),                      # M row 3 on its ref
                   dict(msgs=(1 << 26) + 4 * 2000),                          # in-node rows on its dst rows
                   dict(msgs=(1 << 27) - 4 * 10),                            # ... on its M row 0
                   dict(ref=(1 << 16) + 4 * 50, msgs=1 << 28)):              # ref on its in-node row 0
        arr = (L.MomentumJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_momentum_mix(arr, 2, None) == -1, second
    assert lib.rcmarl_momentum_mix(None, 1, None) == -1
    arr = (L.MomentumJob * 33)(*[_job(dst=(1 << 24) + 4 * 4000 * i, momentum=(1 << 23) + 4 * 2000 * i)
                                 for i in range(33)])
    assert lib.rcmarl_momentum_mix(arr, 0, None) == -1
    assert lib.rcmarl_momentum_mix(arr, 33, None) == -1


def test_check_momentum_refuses_what_the_library_refuses():
    from rcmarl import _lib as L
    for beta in (0, 0.0, 0.5, 0.9, 0.99, np.float32(0.9), np.float64(0.25), 1 - 2 ** -24, 1e-45):
        assert L.check_momentum(beta) == float(beta)
    for beta in (1, 1.0, 1 - 2 ** -26, 1.5, -0.1, -1, float("inf"), float("nan"), "0.9", None, True, [0.9], 1e400):
        with pytest.raises(L.RcmarlError):
            L.check_momentum(beta)


# ------------------------------------------------------------------------------------------------ Trainer
def trainer(momentum, mixing=None, aggregation="clip", H=1, labels=None, attack=None):
    from rcmarl.trainer import Trainer
    return Trainer(labels=labels or MAL, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing, momentum=momentum)


def built(excinfo):
    tb = excinfo.tb
    while tb is not None:
        if tb.tb_frame.f_code.co_name == "__init__" and "momentum" in tb.tb_frame.f_locals:
            return tb.tb_frame.f_locals["self"]
        tb = tb.tb_next
    raise AssertionError("no Trainer frame")


@pytest.mark.parametrize("momentum,mixing,aggregation,labels,attack,match", [
    (1.0, None, "clip", None, None, r"beta in \[0, 1\)"),
    (-0.5, None, "clip", None, None, r"beta in \[0, 1\)"),
    (float("nan"), None, "clip", None, None, r"beta in \[0, 1\)"),
    ([None, None, None, None, 2.0], None, "clip", None, None, r"beta in \[0, 1\)"),     # checked at any agent
    ([0.9, None, "0.5", None, None], None, "clip", None, None, r"beta in \[0, 1\)"),
    ([0.9, 0.9], None, "clip", None, None, "one entry per agent"),
    (0.9, "nnm", "clip", None, None, "both momentum and mixing"),
    ([None, 0.9, None, None, None], [None, ("bucket", 2), None, None, None], "clip", None, None, "agent 1 takes both"),
    (0.9, None, "clip", BYZ, ("tailored_std", 2.0), "whose momentum the attack does not model"),
    ([None, 0.5, None, None, None], None, "scclip", BYZ, ("pipeline_uv", 1.0), "pipeline attack against agent 1"),
])
def test_trainer_refuses_before_any_device_work(no_device, momentum, mixing, aggregation, labels, attack, match):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match=match):
        trainer(momentum, mixing, aggregation, 1, labels, attack)


@pytest.mark.parametrize("momentum,mixing,aggregation,labels,attack", [
    (0.9, None, "clip", None, None), (0.0, None, "krum", None, None), (np.float32(0.99), None, "dnc", None, None),
    (0.9, None, ["mda", "scclip", "gmed", "mkrum", "clip"], BYZ, ("mimic", 5)),
    (0.5, None, "trim", BYZ, ("minsum_uv", 1.0)),
    ([0.9, None, 0.99, None, None], [None, "nnm", None, ("bucket", 2), None], "clip", BYZ, ("dissensus", 1.0)),
    ([0.9, None, None, None, None], None, "clip", BYZ, ("tailored_std", 2.0)),   # agent 0 does not hear agent 4
    ([0.9, None, None, None, None], None, "clip", BYZ, ("pipeline_std", 2.0)),   # agent 0 does not hear agent 4
    ([None, None, None, None, 0.9], "nnm", "clip", None, None),                 # a Malicious agent's beta is ignored
])
def test_trainer_accepts_momentum_alone_and_mixed(no_device, momentum, mixing, aggregation, labels, attack):
    with pytest.raises(no_device):
        trainer(momentum, mixing, aggregation, 1, labels, attack)


def test_trainer_row_layout(no_device):
    """The momentum rows, n_in per agent in mom_agents order, follow every other row block; _rule_nodes returns them."""
    with pytest.raises(no_device) as ex:
        trainer([0.9, None, 0.5, 0.99, 0.7], [None, "nnm", None, None, None], ["scclip", "clip", "dnc", "clip", "clip"],
                1, BYZ, ("gauss", 0.3))
    tr = built(ex)
    assert [p[:2] for p in tr.byz_pairs] == [(4, 1), (4, 2), (4, 3)]
    assert tr.vec_row == {0: 8} and tr.dnc_row == {2: 9} and tr.mix_row == {1: 10}
    assert tr.momentum == [0.9, None, 0.5, 0.99, None] and tr.mom_agents == [0, 2, 3]
    assert tr.mom_row == {0: 14, 2: 18, 3: 22}
    assert tr._rule_nodes(0) == [14, 15, 16, 17] and tr._rule_nodes(2) == [18, 19, 20, 21]
    assert tr._rule_nodes(3) == [22, 23, 24, 25] and tr._rule_nodes(1) == [10, 11, 12, 13]
    assert tr._receiver_nodes(2) == [2, 3, 6, 0]
    with pytest.raises(no_device) as ex:
        trainer(None, None, "clip", 1, BYZ, ("alie", 1.0))
    tr = built(ex)
    assert tr.momentum == [None] * 5 and tr.mom_agents == [] and tr.mom_row == {}
    assert tr._rule_nodes(1) == tr._receiver_nodes(1)


def test_build_trainer_forwards_each_agents_momentum(no_device):
    """train_RPBCAC builds its Trainer with momentum=[agent.momentum]; an adversary has no such attribute."""
    from training.train_agents import build_trainer

    def agent(momentum, H=1):
        return types.SimpleNamespace(get_parameters=lambda: [], H=H, aggregation="clip", mixing=None, momentum=momentum)
    env = types.SimpleNamespace(std_state=1, mean_state=0, randomize_state=True, desired_state=np.zeros((5, 2)),
                                n_envs=4, nrow=5, ncol=5)
    args = dict(agent_label=MAL, in_nodes=C5, gamma=0.9, max_ep_len=10, n_ep_fixed=4, n_epochs=2, buffer_size=100,
                common_reward=False, random_seed=3)
    agents = [agent(0.9), agent(None), agent(0.5), agent(None), types.SimpleNamespace(get_parameters=lambda: [], H=0)]
    with pytest.raises(no_device) as ex:
        build_trainer(env, agents, args)
    tr = built(ex)
    assert tr.momentum == [0.9, None, 0.5, None, None] and tr.mom_agents == [0, 2]
    with pytest.raises(no_device) as ex:
        build_trainer(env, [agent(None) for _ in range(4)] + [agents[-1]], args)
    assert built(ex).mom_agents == []


def test_agent_refuses_bad_momentum_before_touching_its_models():
    """RPBCAC_agent checks beta, and momentum beside mixing, before it reads its models (stand-ins here)."""
    from rcmarl import _lib as L
    from agents.resilient_CAC_agents import RPBCAC_agent
    m = types.SimpleNamespace()
    for kw, match in ((dict(momentum=1.0), r"\[0, 1\)"), (dict(momentum=-0.1), r"\[0, 1\)"),
                      (dict(momentum="0.9"), r"\[0, 1\)"), (dict(momentum=0.9, mixing="nnm"), "momentum and mixing"),
                      (dict(momentum=0.9, mixing=("bucket", 2)), "momentum and mixing")):
        with pytest.raises(L.RcmarlError, match=match):
            RPBCAC_agent(m, m, m, 0.002, 0.01, H=1, **kw)
