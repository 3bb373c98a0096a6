"""CPU checks of the momentum-aware Byzantine messages (rcmarl_history_attack, include/rcmarl.h): the oracle
(tests/history_attack_oracle.py) against pipeline_attack_oracle at c = 0 and first = 1, the modelled rows against
momentum_oracle.step of the messages sent, colluders modelled with their own states, and the inversion; the struct and
symbol as gcc sees the header and the bindings declare them, the library's refusals without a device, the attack
names, the Trainer's refusals and pair layout before it touches a device, and the job tables it builds for its
history pairs."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import adaptive_attack_oracle as AA
import history_attack_oracle as HO
import momentum_oracle as MO
import pipeline_attack_oracle as PA
import tailored_attack_oracle as TA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _stack(rs, n_rows=12, P=40, dtype=f32):
    centre = rs.randn(P)
    X = centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))
    X[-2:] += rs.randn(2, P) * 3.0
    return X.astype(dtype)


# slot 6 a Malicious-style real slot; message 3 sits in slots 2 and 7
SLOTS, HONEST = [0, -1, 3, 4, -1, 5, 10, 3], [0, 2, 3, 5, 7]


@pytest.mark.parametrize("rule", PA.RULES)
@pytest.mark.parametrize("dtype", [np.float64, f32])
def test_at_c_zero_and_first_step_the_oracle_is_the_pipeline_oracle(rule, dtype):
    rs = np.random.RandomState(9100 + len(rule))
    X = _stack(rs, dtype=dtype)
    X[X == 0] = dtype(1)                                  # no -0 anywhere
    c = np.zeros(X.shape[1], dtype)
    for d in ("uv", "std", "sgn"):
        m, g, O, R, rows = HO.craft(X, SLOTS, HONEST, rule, 1, "history_" + d, 2.0, c, None, 0.9, True, [1, 4])
        pm, pg, pO, pR = PA.craft(X, SLOTS, HONEST, rule, 1, "pipeline_" + d, 2.0)
        assert np.array_equal(m, pm) and g == pg and np.array_equal(O, pO) and np.array_equal(R, pR)
        assert np.array_equal(rows[[0, 2, 3, 5, 6, 7]], X[[0, 3, 4, 5, 10, 3]])


@pytest.mark.parametrize("beta", [0.0, 0.5, 0.9, 0.99])
def test_an_own_slot_row_is_the_receivers_step_of_the_sent_message(beta):
    rs = np.random.RandomState(9200)
    X = _stack(rs)
    c = (X[0] + rs.randn(X.shape[1]) * 0.1).astype(f32)
    M = (rs.randn(len(SLOTS), X.shape[1]) * 0.2).astype(f32)
    for rule in ("clip", "gmed", "dnc"):
        m, g, O, R, rows = HO.craft(X, SLOTS, HONEST, rule, 1, "history_std", 2.0, c, M, beta, False, [1, 4])
        sent = np.stack([m if s < 0 else X[s] for s in SLOTS])
        want, _ = MO.step(sent, c, M[:len(SLOTS)], beta, False)            # the receiver's momentum_mix
        assert np.array_equal(rows, want), rule
        assert beta == 0.0 or not np.array_equal(rows[2], rows[7])      # one message, two slots, two states
        assert np.array_equal(R, PA.rule_output(want, rule, 1)), rule
        assert np.isfinite(O).any() and g >= 0


def test_colluders_are_modelled_with_their_own_states():
    """Own slot 1 and colluder slot 4: the colluder's modelled message inverts the same target with M_4, and all own
    slots share the inversion with M_1 (the lowest own slot)."""
    rs = np.random.RandomState(9300)
    X = _stack(rs)
    c = (X[0] * 0.5).astype(f32)
    M = (rs.randn(len(SLOTS), X.shape[1]) * 0.3).astype(f32)
    beta = 0.9
    m, g, O, R, rows = HO.craft(X, SLOTS, HONEST, "trim", 1, "history_uv", 2.0, c, M, beta, False, [1])
    mu, d, _ = AA.gamma_of(rows[HONEST], "minmax_uv")
    t = TA.candidate(mu, d, g)                            # the target gamma_i* steers every crafted row to
    assert np.array_equal(m, HO.invert(t, c, M[1], beta, False))
    assert np.array_equal(rows[1], HO.step_row(m, c, M[1], beta, False))
    assert np.array_equal(rows[4], HO.step_row(HO.invert(t, c, M[4], beta, False), c, M[4], beta, False))
    np.testing.assert_allclose(rows[[1, 4]], np.stack([t, t]), rtol=1e-5, atol=1e-5)
    # the same job with both crafted slots own: slot 4 then receives M_1's inversion
    m2, g2, _, _, rows2 = HO.craft(X, SLOTS, HONEST, "trim", 1, "history_uv", 2.0, c, M, beta, False, [4, 1])
    t2 = TA.candidate(mu, d, g2)
    assert np.array_equal(m2, HO.invert(t2, c, M[1], beta, False))
    assert np.array_equal(rows2[4], HO.step_row(m2, c, M[4], beta, False))
    assert np.abs(rows2[4] - t2).max() > 1e-3            # M_4 differs from M_1, so the row misses the target


def test_the_inversion_restated():
    f = f32
    t, c, M = np.array([1.0, 2.0, -3.0, 5.0], f), np.array([0.5, 0.0, 1.0, 2.0], f), np.array([0.25, np.inf, -1.0, -np.inf], f)
    got = HO.invert(t, c, M, 0.5, False)
    b = f(0.5)
    want0 = f(c[0] + f(f(f(t[0] - c[0]) - f(b * M[0])) / f(f(1) - b)))
    assert got[0] == want0 and got[1] == t[1] and got[3] == t[3]
    assert np.array_equal(HO.invert(t, c, M, 0.5, True), t)
    # one step of the momentum row of the inverted message lands on t up to the step's own roundings
    r = HO.step_row(got, c, M, 0.5, False)
    np.testing.assert_allclose(r[[0, 2]], t[[0, 2]], rtol=1e-6)
    assert np.isinf(HO.invert(np.array([3e38], f), np.array([-3e38], f), np.array([0.0], f), 0.99, False)[0])


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_struct_constant_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = [f[0] for f in L.HistoryAttackJob._fields_]
    assert fields == ["attack", "model_out", "ref", "momentum", "momentum_stride", "beta", "first", "own_mask",
                      "reserved"]
    offs = " ".join(f'printf("%d ", (int)offsetof(rcmarl_history_attack_job, {f}));' for f in fields)
    src = tmp_path / "hist.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_history_attack_job*, int, void*) = rcmarl_history_attack; (void)f;'
                   'printf("%d %d %d ", RCMARL_HISTORY_MAX_FLOATS, (int)RCMARL_TAILOR_SPECTRAL,'
                   f'(int)sizeof(rcmarl_history_attack_job)); {offs} return 0;}}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_history_attack(const rcmarl_history_attack_job* j, int n, '
                    'void* s){(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "hist"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[:2] == [L.HISTORY_MAX_FLOATS, L.TAILOR_SPECTRAL] == [22 * 1421, 2]
    assert got[2] == ctypes.sizeof(L.HistoryAttackJob)
    assert got[3:] == [getattr(L.HistoryAttackJob, f).offset for f in fields]
    assert L.lib().rcmarl_history_attack.argtypes == [ctypes.POINTER(L.HistoryAttackJob), ctypes.c_int, L.c_fp]
    assert ("rcmarl_history_attack", ctypes.c_int, [ctypes.POINTER(L.HistoryAttackJob), ctypes.c_int, L.c_fp]) \
        in L.SYMBOLS


def test_staging_bound_is_the_16_agent_team_reward_net_under_dnc():
    from rcmarl import _lib as L
    P = L.param_count(48, 1)
    assert P == 1421 and (16 + 4 + 2) * P == L.HISTORY_MAX_FLOATS == HO.MAX_FLOATS
    assert L.HISTORY_MAX_FLOATS * 4 + 8 * 1024 <= 227 * 1024


def _job(**kw):
    """A valid job on made-up addresses: a C2 receiver (slots 0, 1, crafted, 3) of 100-float rows 1000 floats apart,
    clip H = 1; M rows 1000 floats apart at 1 << 20, ref at 1 << 22; dst, gamma_out and model_out far away."""
    from rcmarl import _lib as L
    j = L.HistoryAttackJob()
    a = j.attack
    a.dst, a.msgs, a.msg_stride, a.n, a.n_in = 1 << 24, 1 << 16, 1000, 100, 4
    a.gamma_out = (1 << 24) + 4 * 200
    for k, v in enumerate([0, 1, -1, 3]):
        a.slots[k] = v
    a.honest_mask, a.family, a.rule, a.H, a.dev, a.scale = 0b1011, L.TAILOR_COORD, L.AGG_CLIP, 1, L.DEV_STD, 2.0
    j.model_out = (1 << 24) + 4 * 400
    j.ref, j.momentum, j.momentum_stride, j.beta, j.first, j.own_mask = 1 << 22, 1 << 20, 1000, 0.9, 0, 0b0100
    for k, v in kw.items():
        if k == "slots":
            for i, x in enumerate(v):
                a.slots[i] = x
        elif k in ("model_out", "ref", "momentum", "momentum_stride", "beta", "first", "own_mask"):
            setattr(j, k, v)
        else:
            setattr(a, k, v)
    return j


BAD = [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n_in=0), dict(n_in=17), dict(honest_mask=0b10011),
    dict(slots=[0, 1, 2, 3], own_mask=0), dict(honest_mask=0), dict(honest_mask=0b0111), dict(slots=[0, 1, -2, 3]),
    dict(family=3), dict(rule=3), dict(family=1, rule=4), dict(family=2, rule=1), dict(dev=3), dict(dev=-1),
    dict(scale=-1.0), dict(scale=float("nan")), dict(scale=float("inf")), dict(H=-1), dict(H=4),
    dict(family=1, rule=0, H=2),                                          # krum at n_in = 4 < H + 3
    dict(ref=None), dict(momentum=None),
    dict(beta=1.0), dict(beta=-0.5), dict(beta=float("nan")), dict(beta=float("inf")), dict(first=2), dict(first=-1),
    dict(own_mask=0), dict(own_mask=0b0101), dict(own_mask=0b10100),      # empty, on a real slot, past n_in
    dict(n=22 * 1421 // 8 + 1),                                           # staging: (4 + 4) * n > bound
    dict(dst=(1 << 16) + 4 * 1000),                                       # dst on slot 1's row
    dict(gamma_out=(1 << 16) + 4 * 3050),                                 # gamma_out on slot 3's row
    dict(model_out=(1 << 16) + 4 * 10),                                   # model_out on slot 0's row
    dict(model_out=(1 << 24) + 4 * 50),                                   # ... on the job's dst
    dict(dst=(1 << 22) + 4 * 50),                                         # dst on the ref
    dict(model_out=(1 << 20) + 4 * 3050),                                 # model_out on M row 3
    dict(gamma_out=(1 << 20) + 4 * 2000),                                 # gamma_out on M row 2 (a crafted slot's)
]


@pytest.mark.parametrize("bad", BAD)
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    other = _job(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000)
    for jobs in ([_job(**bad)], [other, _job(**bad)]):
        arr = (L.HistoryAttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_history_attack(arr, len(arr), None) == -1, bad     # RCMARL_ERR_ARG


def test_one_float_past_the_staging_bound_is_refused_without_a_device():
    """DnC at n_in = 16 with one crafted slot: (16 + 4 + 2) * 1422 floats is one row of floats past the bound (the
    1421-parameter job at the bound itself runs in tests/test_history_attack_gpu.py)."""
    from rcmarl import _lib as L
    lib = L.lib()
    j = _job(n=1422, n_in=16, slots=list(range(15)) + [-1], honest_mask=(1 << 15) - 1, family=L.TAILOR_SPECTRAL,
             rule=L.SPECTRAL_DNC, H=3, msg_stride=2000, momentum_stride=2000, dst=1 << 28, gamma_out=1 << 27,
             model_out=(1 << 27) + 64, own_mask=1 << 15)
    assert lib.rcmarl_history_attack((L.HistoryAttackJob * 1)(j), 1, None) == -1


def test_library_refuses_bad_job_counts_and_cross_job_overlaps_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_history_attack(None, 1, None) == -1
    arr = (L.HistoryAttackJob * 33)(*[_job(dst=(1 << 26) + 4 * 1000 * i, gamma_out=(1 << 27) + 4 * i,
                                           model_out=(1 << 28) + 4 * 1000 * i) for i in range(33)])
    assert lib.rcmarl_history_attack(arr, 0, None) == -1
    assert lib.rcmarl_history_attack(arr, 33, None) == -1
    first = dict(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000)
    for second in (dict(model_out=(1 << 26) + 4 * 50), dict(model_out=(1 << 26) + 4 * 8000),
                   dict(dst=(1 << 26) + 4 * 9050), dict(model_out=(1 << 26) + 4 * 9099)):
        arr = (L.HistoryAttackJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_history_attack(arr, 2, None) == -1, second
    for other in (dict(ref=(1 << 28) + 4 * 50), dict(momentum=1 << 28)):      # the other job's ref / M rows
        arr = (L.HistoryAttackJob * 2)(_job(**other), _job(model_out=(1 << 28) + 4 * 10))
        assert lib.rcmarl_history_attack(arr, 2, None) == -1, other


def test_attack_names_and_bindings():
    import torch
    from rcmarl import _lib as L, ops
    for d, dev in (("uv", 0), ("std", 1), ("sgn", 2)):
        kind, param = L.check_attack((f"history_{d}", 2))
        assert isinstance(kind, L.HistoryKind) and int(kind) == dev and param == 2.0
        assert not isinstance(kind, (L.PipelineKind, L.TailoredKind))
        assert L.is_history_attack(f"history_{d}") and not L.is_pipeline_attack(f"history_{d}")
    for bad in (("history_uv", -0.5), ("history_std", float("nan")), ("history_sgn", float("inf")), ("history", 1.0),
                ("history_dnc", 1.0)):
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)
    x = torch.zeros(8, 50)
    M = torch.zeros(4, 60)
    j = ops.history_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "dnc", 1, "history_sgn", 1.5, x[6], M, 60,
                               0.9, 1, [2], gamma_out=x[4, :1], model_out=x[7])
    assert (j.attack.family, j.attack.rule, j.attack.H, j.attack.dev) == (L.TAILOR_SPECTRAL, L.SPECTRAL_DNC, 1, 2)
    assert j.attack.honest_mask == 0b1011 and list(j.attack.slots[:4]) == [0, 1, -1, 3] and j.attack.scale == 1.5
    assert (j.ref, j.momentum, j.momentum_stride, j.first, j.own_mask) == (x[6].data_ptr(), M.data_ptr(), 60, 1, 4)
    assert abs(j.beta - 0.9) < 1e-7 and j.model_out == x[7].data_ptr() and j.attack.gamma_out == x[4].data_ptr()
    assert ops.history_attack_job(x[5], x, 50, 50, [0, -1], [0], "gmed", 0, "history_uv", 1.0, x[6], M, 60, 0.5, 0,
                                  [1]).attack.family == L.TAILOR_VECTOR
    for bad in (dict(attack="pipeline_uv"), dict(rule="median"), dict(own=[4]), dict(own=[-1])):
        args = dict(rule="clip", attack="history_uv", own=[1])
        args.update(bad)
        with pytest.raises(L.RcmarlError):
            ops.history_attack_job(x[5], x, 50, 50, [0, -1], [0], args["rule"], 0, args["attack"], 1.0, x[6], M, 60,
                                   0.5, 0, args["own"])


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


def trainer(aggregation, momentum, attack=("history_std", 2.0), mixing=None, H=1):
    from rcmarl.trainer import Trainer
    return Trainer(labels=BYZ, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing, momentum=momentum)


def built(excinfo):
    tb = excinfo.tb
    while tb is not None:
        if tb.tb_frame.f_code.co_name == "__init__" and "momentum" in tb.tb_frame.f_locals:
            return tb.tb_frame.f_locals["self"]
        tb = tb.tb_next
    raise AssertionError("no Trainer frame")


@pytest.mark.parametrize("aggregation,momentum,mixing", [
    ("clip", 0.9, None), ("dnc", 0.99, None), ("gmed", [0.9, None, 0.5, None, None], None),
    (["krum", "trim", "scclip", "dnc", "clip"], [None, 0.9, None, 0.9, None], [None, None, "nnm", None, None]),
    ("wmsr", None, "bucket"),
])
def test_trainer_accepts_history_attackers_against_every_rule_with_and_without_momentum(no_device, aggregation,
                                                                                          momentum, mixing):
    for attack in (("history_std", 2.0), ("history_uv", 1.0), ("history_sgn", 0.0)):
        with pytest.raises(no_device) as ex:
            trainer(aggregation, momentum, attack=attack, mixing=mixing)
        tr = built(ex)
        assert tr.hist_pairs == [0, 1, 2] and tr.pipe_pairs == [] and tr.gamma_pairs == [0, 1, 2]


@pytest.mark.parametrize("rule", ["mda", "smea"])
@pytest.mark.parametrize("momentum", [None, 0.9])
def test_trainer_refuses_history_attacks_against_subset_rules(no_device, rule, momentum):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match=f"history attack against agent .*'{rule}' the attack does not model"):
        trainer(rule, momentum)


@pytest.mark.parametrize("s", [-1.0, float("nan"), float("inf")])
def test_trainer_refuses_a_bad_scale(no_device, s):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="needs a finite parameter"):
        trainer("clip", 0.9, attack=("history_uv", s))


@pytest.mark.parametrize("name", ["pipeline_std", "tailored_uv"])
def test_pipeline_and_tailored_attacks_stay_refused_against_momentum(no_device, name):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="whose momentum the attack does not model"):
        trainer("clip", 0.9, attack=(name, 2.0))


def test_history_pairs_follow_the_pipeline_pairs_in_gamma_pairs(no_device):
    from rcmarl import _lib as L
    from rcmarl.trainer import Trainer
    labels = ["Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative",
              "Byzantine"]
    in_nodes = [[i, (i + 1) % 8, (i + 2) % 8, (i + 3) % 8] for i in range(8)]
    attack = [None, ("history_uv", 1.0), None, ("minmax_std", 1.0), None, ("pipeline_sgn", 2.0), None,
              ("tailored_std", 2.0)]
    with pytest.raises(no_device) as ex:
        Trainer(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((8, 2)), H=1, attack=attack)
    tr = built(ex)
    assert tr.gamma_pairs == tr.adapt_pairs + tr.tailor_pairs + tr.pipe_pairs + tr.hist_pairs
    assert tr.hist_pairs and {tr.byz_pairs[e][0] for e in tr.hist_pairs} == {1}
    assert all(isinstance(tr.attack[tr.byz_pairs[e][0]][0], L.HistoryKind) for e in tr.hist_pairs)


def test_job_layout_of_a_trainer_with_momentum_and_plain_receivers(monkeypatch):
    """Two history attackers (agent 4 listed twice by receiver 2), receivers 2 and 3 with momentum and receiver 1
    without: the history jobs' fields, hist_mom, and the pipeline jobs of the receiver without momentum, built on host
    tensors (the job tables only take pointers)."""
    import torch
    from rcmarl import _lib as L, ops
    from rcmarl.trainer import Trainer
    monkeypatch.setattr(ops, "workspace", lambda *a, **k: torch.zeros(8, dtype=torch.uint8))
    labels = ["Cooperative"] * 4 + ["Byzantine"] * 2
    in_nodes = [[0, 1, 2, 3], [1, 2, 4, 5], [2, 4, 3, 4, 5], [3, 0, 5, 1], [4, 0, 1, 2], [5, 0, 1, 2]]
    mom = [0.9, None, 0.99, 0.5, None, None]
    tr = Trainer(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((6, 2)), H=1, device="cpu",
                 attack=[None] * 4 + [("history_std", 2.0), ("history_uv", 1.0)], momentum=mom)
    assert tr.byz_pairs == [(4, 1, [1, 2]), (4, 2, [2, 3]), (5, 1, [1, 2]), (5, 2, [2, 3]), (5, 3, [3, 0, 1])]
    assert tr.hist_pairs == [0, 1, 2, 3, 4] and tr.gamma_pairs == tr.hist_pairs and tr.mom_agents == [0, 2, 3]
    att, ada, tail, pipe, hist, hist_mom, diss, _, mimic = tr._attack_job_groups()
    assert att == ada == tail == diss == mimic == [] and len(pipe) == 1 and len(hist) == 1 and hist[0][0] == 0
    assert hist_mom == [1, 1, 1, 1, 2, 2]
    NA = tr.NA
    want = {1: (2, [0, -1, 2, -1, -1], 0b00101, 0b01010, L.DEV_STD, 2.0),
            3: (2, [0, -1, 2, -1, -1], 0b00101, 0b10000, L.DEV_UV, 1.0),
            4: (3, [3, 0, -1, 1], 0b1011, 0b0100, L.DEV_UV, 1.0)}
    jobs = list(hist[0][1])
    assert all(isinstance(j, L.HistoryAttackJob) for j in jobs) and len(jobs) == 6
    for n, (e, t) in enumerate((e, t) for e in (1, 3, 4) for t in (0, 1)):
        j, (r, slots, honest_mask, own_mask, dev, scale) = jobs[n], want[e]
        msgs, P, ref = (tr.msg_c, tr.PC, tr.critic[r]) if t == 0 else (tr.msg_t, tr.PT, tr.tr[r])
        a = j.attack
        assert (a.dst, a.msgs, a.msg_stride, a.n, a.n_in) == (msgs[NA + e].data_ptr(), msgs.data_ptr(), P, P, len(slots))
        slots = [s if s < 0 else in_nodes[r][k] for k, s in enumerate(slots)]
        assert list(a.slots[:a.n_in]) == slots and a.honest_mask == honest_mask
        assert (a.family, a.rule, a.H, a.dev, a.scale) == (L.TAILOR_COORD, L.AGG_CLIP, 1, dev, scale)
        assert a.gamma_out == tr.att_gamma[tr.gamma_pairs.index(e), t:t + 1].data_ptr() and j.model_out is None
        q = tr.mom_agents.index(r)
        assert (j.ref, j.momentum, j.momentum_stride) == (ref.data_ptr(), tr.momentum_M[q, t].data_ptr(), tr.PT)
        assert j.beta == np.float32(mom[r]) and j.first == 0 and j.own_mask == own_mask
    pj = list(pipe[0])
    assert all(isinstance(j, L.PipelineAttackJob) for j in pj) and len(pj) == 4
    for j, (e, t) in zip(pj, ((0, 0), (0, 1), (2, 0), (2, 1))):
        msgs, P = (tr.msg_c, tr.PC) if t == 0 else (tr.msg_t, tr.PT)
        a = j.attack
        assert (a.dst, a.n, list(a.slots[:4]), a.honest_mask) == (msgs[NA + e].data_ptr(), P, [1, 2, -1, -1], 0b11)
        assert (a.dev, a.scale) == ((L.DEV_STD, 2.0) if e == 0 else (L.DEV_UV, 1.0))
        assert j.mixing == L.PIPE_NONE and a.gamma_out == tr.att_gamma[tr.gamma_pairs.index(e), t:t + 1].data_ptr()
        assert (j.attacker, j.receiver, j.net) == (tr.byz_pairs[e][0], 1, t)
