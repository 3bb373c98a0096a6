"""CPU checks of the pipeline-aware Byzantine messages (rcmarl_pipeline_attack, include/rcmarl.h): the oracle
(tests/pipeline_attack_oracle.py) against tailored_attack_oracle without mixing, nnm at H = n_in - 1 and scale 0, the
Philox counter words of the attacker's shuffle samples, the enums and struct as gcc sees the header and the bindings
declare them, the library's refusals without a device, the attack names, and the Trainer's acceptance and pair layout
before it touches a device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import adaptive_attack_oracle as AA
import attack_oracle as AT
import bucket_oracle as BO
import pipeline_attack_oracle as PA
import tailored_attack_oracle as TA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stack(rs, n_rows=12, P=40, dtype=np.float64):
    centre = rs.randn(P)
    X = centre + rs.randn(n_rows, P) * rs.uniform(0.05, 1.0, size=(n_rows, 1))
    X[-2:] += rs.randn(2, P) * 3.0
    return X.astype(dtype)


def _case(rs, n_in, n_rows=12):
    n_cr = 1 + rs.randint(min(3, n_in - 1))
    real = [int(x) for x in rs.choice(n_rows, size=n_in - n_cr, replace=False)]
    slots = real[:1] + [-1] * n_cr + real[1:]
    rs.shuffle(slots[1:])
    honest = [k for k, s in enumerate(slots) if s >= 0 and s < n_rows - 2]
    return slots, honest or [0]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("rule", TA.RULES)
def test_without_mixing_the_oracle_is_the_tailored_oracle(dtype, rule):
    rs = np.random.RandomState(7100 + len(rule))
    X = _stack(rs, dtype=dtype)
    for n_in in (3, 5, 8):
        slots, honest = _case(rs, n_in)
        if slots[0] < 0 or slots[0] >= 10:
            continue
        H = 0 if rule in ("krum", "mkrum") and n_in < 4 else 1
        for d in AA.DEVS:
            want = TA.craft(X, slots, honest, rule, H, "tailored_" + d, 2.0)
            got = PA.craft(X, slots, honest, rule, H, "pipeline_" + d, 2.0)
            assert np.array_equal(got[0], want[0]) and got[1] == want[1]
            assert np.array_equal(got[2], want[2])


@pytest.mark.parametrize("rule", PA.RULES)
def test_nnm_at_H_n_in_minus_1_is_no_mixing(rule):
    """nnm at H = n - 1 passes every row through, so the attack is the unmixed one at that H."""
    rs = np.random.RandomState(7200)
    X = _stack(rs)
    for n_in in (4, 6):
        slots, honest = _case(rs, n_in)
        H = n_in - 1
        if rule in ("krum", "mkrum", "trim"):
            continue                                      # these rules refuse H = n - 1
        a = PA.craft(X, slots, honest, rule, H, "pipeline_std", 2.0, mixing="nnm")
        b = PA.craft(X, slots, honest, rule, H, "pipeline_std", 2.0)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])
        assert np.array_equal(a[3], b[3])


@pytest.mark.parametrize("mixing", [None, "nnm", ("bucket", 2), ("bucket", 3)])
@pytest.mark.parametrize("rule", ["clip", "gmed", "dnc"])
def test_scale_zero_gives_mu(mixing, rule):
    rs = np.random.RandomState(7300)
    X = _stack(rs)
    slots, honest = [0, -1, 3, 4, -1, 5], [0, 2, 3, 5]
    msg, g, Ob, R = PA.craft(X, slots, honest, rule, 1, "pipeline_uv", 0.0, mixing=mixing, n_perms=3, seed=5,
                             attacker=4, receiver=2, net=1, round_=9, epoch=1)
    mu = AA.gamma_of(X[[0, 3, 4, 5]], "minmax_uv")[0]
    assert g == 0 and np.array_equal(msg, mu) and np.isfinite(Ob).all() and len(set(Ob.tolist())) == 1


def test_counter_words_and_stream_separation():
    assert PA.counter(0, 0, 0, 0, 0, 0, 0) == (0, 0x10000000, 0, 0)
    assert PA.counter(3, 9, 4, 2, 1, 7, 5) == (3 << 2 | 2, 4 | 2 << 8 | 1 << 16 | 0x10000000, 7, 5)
    assert PA.counter(15, 14, 255, 255, 1, 2 ** 32 + 3, 1) == (63, 255 | 255 << 8 | 1 << 16 | 0x10000000, 3, 1)
    for q in range(16):
        for t in range(14):                            # at most 14 draws (n_in = 16)
            w0, w1 = PA.counter(q, t, 255, 255, 1, 0, 0)[:2]
            assert w0 >> 2 == q and w0 & 3 == t >> 2
            assert w1 & 0xF0000000 == 0x10000000         # bit 28 alone of the top four: no other stream's word 1
    a = PA.draws(14, 7, 0, 4, 2, 1, 3, 0)
    assert len(set(a)) == 14
    for kw in (dict(q=1), dict(attacker=3), dict(receiver=1), dict(net=0), dict(round_=4), dict(epoch=1), dict(seed=8)):
        args = dict(seed=7, q=0, attacker=4, receiver=2, net=1, round_=3, epoch=0)
        args.update(kw)
        assert PA.draws(14, **args) != a, kw
    # the same Philox words, read through attack_oracle directly
    ctr = [np.array([PA.counter(2, 0, 4, 2, 1, 3, 0)[w]], np.uint64) for w in range(4)]
    words = AT.philox4x32_10(ctr, (7, 0))
    assert PA.draws(4, 7, 2, 4, 2, 1, 3, 0) == [int(words[w][0]) for w in range(4)]
    for n_in in range(2, 17):
        for s in (1, 2, 3, 16):
            bks = PA.buckets(n_in, s, 11, 3, 1, 2, 0, 5, 6)
            assert sorted(sum(bks, [])) == list(range(1, n_in)) and len(bks) == BO.n_out(n_in, s) - 1


def test_the_mean_objective_averages_the_samples_in_q_order():
    """Obar_i = (O_i,0 + O_i,1 + O_i,2) / 3 in fp32, each O_i,q from sample q's buckets."""
    rs = np.random.RandomState(7400)
    X = _stack(rs, dtype=np.float32)
    slots, honest = [0, 1, -1, 2, 3, 4, -1, 5], [0, 1, 3, 4, 5]
    words = dict(seed=3, attacker=6, receiver=0, net=0, round_=2, epoch=1)
    msg, g, Ob, R = PA.craft(X, slots, honest, "trim", 1, "pipeline_std", 2.0, mixing=("bucket", 2), n_perms=3, **words)
    assert Ob.dtype == np.float32 and np.isfinite(Ob).all()
    V = X[[0, 1, 2, 3, 4]]
    mu, d, g_mm = AA.gamma_of(V, "minmax_std")
    bks = [PA.buckets(8, 2, 3, q, 6, 0, 0, 2, 1) for q in range(3)]
    assert bks[0] != bks[1] or bks[1] != bks[2]
    for i in (0, 7, PA.STEPS):
        gi = np.float32(np.float32(np.float32(2.0) * g_mm) * np.float32(i)) / np.float32(PA.STEPS)
        m = TA.candidate(mu, d, gi)
        Xs = np.stack([m if s < 0 else X[s] for s in slots])
        O = [TA.objective(TA.rule_output(BO.mix(Xs, b)[0], "trim", 1), mu) for b in bks]
        assert Ob[i] == np.float32(np.float32(np.float32(np.float32(0) + O[0]) + O[1]) + O[2]) / np.float32(3)
    i = int(np.argmax(Ob))
    assert g == np.float32(np.float32(np.float32(2.0) * g_mm) * np.float32(i)) / np.float32(PA.STEPS)
    Xs = np.stack([msg if s < 0 else X[s] for s in slots])
    assert np.array_equal(R, TA.rule_output(BO.mix(Xs, bks[0])[0], "trim", 1))


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_enums_struct_and_symbol_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = [f[0] for f in L.PipelineAttackJob._fields_]
    assert fields == ["attack", "model_out", "seed", "mixing", "s", "n_perms", "attacker", "receiver", "net", "round",
                      "epoch"]
    offs = " ".join(f'printf("%d ", (int)offsetof(rcmarl_pipeline_attack_job, {f}));' for f in fields)
    src = tmp_path / "pipe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'int (*f)(const rcmarl_pipeline_attack_job*, int, void*) = rcmarl_pipeline_attack; (void)f;'
                   'printf("%d %d %d %d %d %d %d ", (int)RCMARL_PIPE_NONE, (int)RCMARL_PIPE_NNM, (int)RCMARL_PIPE_BUCKET,'
                   '(int)RCMARL_TAILOR_SPECTRAL, RCMARL_PIPELINE_MAX_FLOATS, RCMARL_PIPELINE_MAX_PERMS,'
                   f'(int)sizeof(rcmarl_pipeline_attack_job)); {offs} return 0;}}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\nint rcmarl_pipeline_attack(const rcmarl_pipeline_attack_job* j, int n, '
                    'void* s){(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "pipe"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[:4] == [L.PIPE_NONE, L.PIPE_NNM, L.PIPE_BUCKET, L.TAILOR_SPECTRAL] == [0, 1, 2, 2]
    assert got[4:6] == [L.PIPELINE_MAX_FLOATS, L.PIPELINE_MAX_PERMS] == [37 * 1421, 16]
    assert got[6] == ctypes.sizeof(L.PipelineAttackJob)
    assert got[7:] == [getattr(L.PipelineAttackJob, f).offset for f in fields]
    assert L.PipelineAttackJob.attack.offset == 0 and L.PipelineAttackJob.attack.size == ctypes.sizeof(L.TailoredAttackJob)
    assert L.lib().rcmarl_pipeline_attack.argtypes == [ctypes.POINTER(L.PipelineAttackJob), ctypes.c_int, L.c_fp]


def test_staging_bound_is_the_16_agent_team_reward_net_under_nnm():
    from rcmarl import _lib as L
    P = L.param_count(48, 1)
    assert P == 1421 and (15 + 16 + 4 + 2) * P == L.PIPELINE_MAX_FLOATS
    assert L.PIPELINE_MAX_FLOATS * 4 <= 227 * 1024 - 8 * 1024     # room left for the kernel's static shared memory


def _job(**kw):
    """A valid job on made-up addresses: a C2 receiver (slots 0, 1, crafted, 3) of 100-float rows 1000 floats apart,
    clip H = 1, bucketing at s = 2 with 4 samples; dst, gamma_out and model_out far away."""
    from rcmarl import _lib as L
    j = L.PipelineAttackJob()
    a = j.attack
    a.dst, a.msgs, a.msg_stride, a.n, a.n_in = 1 << 24, 1 << 16, 1000, 100, 4
    a.gamma_out = (1 << 24) + 4 * 200
    for k, v in enumerate([0, 1, -1, 3]):
        a.slots[k] = v
    a.honest_mask, a.family, a.rule, a.H, a.dev, a.scale = 0b1011, L.TAILOR_COORD, L.AGG_CLIP, 1, L.DEV_STD, 2.0
    j.model_out = (1 << 24) + 4 * 400
    j.mixing, j.s, j.n_perms = L.PIPE_BUCKET, 2, 4
    j.seed, j.attacker, j.receiver, j.net, j.round, j.epoch = 5, 4, 1, 1, 9, 2
    for k, v in kw.items():
        if k == "slots":
            for i, x in enumerate(v):
                a.slots[i] = x
        elif k in ("model_out", "seed", "mixing", "s", "n_perms", "attacker", "receiver", "net", "round", "epoch"):
            setattr(j, k, v)
        else:
            setattr(a, k, v)
    return j


BAD = [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n_in=0), dict(n_in=17), dict(honest_mask=0b10011),
    dict(slots=[0, 1, 2, 3]), dict(honest_mask=0), dict(honest_mask=0b0111), dict(slots=[0, 1, -2, 3]),
    dict(family=3), dict(rule=3), dict(family=1, rule=4), dict(family=2, rule=1), dict(dev=3), dict(dev=-1),
    dict(scale=-1.0), dict(scale=float("nan")), dict(scale=float("inf")), dict(H=-1),
    dict(H=3), dict(H=2, mixing=0, rule=1),                               # H >= n_rows = 3 (bucketing); trim 2H >= 4
    dict(family=1, rule=0, H=1),                                          # krum at n_rows = 3 < H + 3
    dict(family=1, rule=1, H=0, mixing=1, n_in=2, slots=[0, -1], honest_mask=1),     # mkrum at n_in 2 < 3
    dict(mixing=3), dict(mixing=-1),
    dict(s=0), dict(s=-2), dict(n_perms=0), dict(n_perms=17), dict(attacker=256), dict(receiver=256), dict(net=2),
    dict(n=37 * 1421 // 9 + 1),                                           # staging: (3 + 2 + 4) * n > bound
    dict(dst=(1 << 16) + 4 * 1000),                                       # dst on slot 1's row
    dict(gamma_out=(1 << 16) + 4 * 3050),                                 # gamma_out on slot 3's row
    dict(model_out=(1 << 16) + 4 * 10),                                   # model_out on slot 0's row
    dict(model_out=(1 << 24) + 4 * 50),                                   # ... on the job's dst
    dict(model_out=(1 << 24) + 4 * 200 - 4 * 99),                         # ... reaching its gamma_out
]


@pytest.mark.parametrize("bad", BAD)
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    for jobs in ([_job(**bad)], [_job(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000),
                                 _job(**bad)]):
        arr = (L.PipelineAttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_pipeline_attack(arr, len(arr), None) == -1, bad     # RCMARL_ERR_ARG


def test_one_float_past_the_staging_bound_is_refused_without_a_device():
    """DnC under nnm at n_in = 16 with one crafted slot: (15 + 16 + 4 + 2) * 1422 floats is one row of floats past
    the bound (the 1421-parameter job at the bound itself runs in tests/test_pipeline_attack_gpu.py)."""
    from rcmarl import _lib as L
    lib = L.lib()
    j = _job(n=1422, n_in=16, slots=list(range(15)) + [-1], honest_mask=(1 << 15) - 1, family=L.TAILOR_SPECTRAL,
             rule=L.SPECTRAL_DNC, H=3, mixing=L.PIPE_NNM, msg_stride=2000, dst=1 << 28, gamma_out=1 << 27,
             model_out=(1 << 27) + 64)
    assert lib.rcmarl_pipeline_attack((L.PipelineAttackJob * 1)(j), 1, None) == -1


def test_tailored_attack_still_refuses_the_spectral_family_and_a_mixing_receiver_is_not_its_concern():
    from rcmarl import _lib as L
    lib = L.lib()
    t = _job(mixing=0).attack
    t.family, t.rule = L.TAILOR_SPECTRAL, L.SPECTRAL_DNC
    assert lib.rcmarl_tailored_attack((L.TailoredAttackJob * 1)(t), 1, None) == -1


def test_library_refuses_bad_job_counts_and_cross_job_overlaps_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_pipeline_attack(None, 1, None) == -1
    arr = (L.PipelineAttackJob * 33)(*[_job(dst=(1 << 26) + 4 * 1000 * i, gamma_out=(1 << 27) + 4 * i,
                                            model_out=(1 << 28) + 4 * 1000 * i) for i in range(33)])
    assert lib.rcmarl_pipeline_attack(arr, 0, None) == -1
    assert lib.rcmarl_pipeline_attack(arr, 33, None) == -1
    first = dict(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000)
    for second in (dict(model_out=(1 << 26) + 4 * 50), dict(model_out=(1 << 26) + 4 * 8000),
                   dict(dst=(1 << 26) + 4 * 9050), dict(model_out=(1 << 26) + 4 * 9099)):
        arr = (L.PipelineAttackJob * 2)(_job(**first), _job(**second))
        assert lib.rcmarl_pipeline_attack(arr, 2, None) == -1, second
    arr = (L.PipelineAttackJob * 2)(_job(msgs=1 << 28), _job(model_out=(1 << 28) + 4 * 3000))
    assert lib.rcmarl_pipeline_attack(arr, 2, None) == -1                  # model_out on the other job's slot row


def test_attack_names_and_bindings():
    import torch
    from rcmarl import _lib as L, ops
    for d, dev in (("uv", 0), ("std", 1), ("sgn", 2)):
        kind, param = L.check_attack((f"pipeline_{d}", 2))
        assert isinstance(kind, L.PipelineKind) and int(kind) == dev and param == 2.0
        assert not isinstance(kind, L.TailoredKind)
    for bad in (("pipeline_uv", -0.5), ("pipeline_std", float("nan")), ("pipeline", 1.0), ("pipeline_dnc", 1.0)):
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)
    x = torch.zeros(6, 50)
    j = ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "dnc", 1, "pipeline_sgn", 1.5,
                                mixing="bucket", n_perms=4, seed=2 ** 40 + 3, attacker=4, receiver=2, net=1, round=7,
                                epoch=3, gamma_out=x[4, :1], model_out=x[4, 1:])
    assert (j.attack.family, j.attack.rule, j.attack.H, j.attack.dev) == (L.TAILOR_SPECTRAL, L.SPECTRAL_DNC, 1, 2)
    assert j.attack.honest_mask == 0b1011 and list(j.attack.slots[:4]) == [0, 1, -1, 3] and j.attack.scale == 1.5
    assert (j.mixing, j.s, j.n_perms, j.seed) == (L.PIPE_BUCKET, 2, 4, 2 ** 40 + 3)
    assert (j.attacker, j.receiver, j.net, j.round, j.epoch) == (4, 2, 1, 7, 3)
    assert j.model_out == x[4, 1:].data_ptr() and j.attack.gamma_out == x[4].data_ptr()
    assert ops.pipeline_attack_job(x[5], x, 50, 50, [0, -1], [0], "gmed", 0, "pipeline_uv", 1.0,
                                   mixing="nnm").attack.family == L.TAILOR_VECTOR
    k = ops.pipeline_attack_job(x[5], x, 50, 50, [0, -1], [0], "trim", 0, "pipeline_uv", 1.0, mixing=("bucket", 3))
    assert (k.mixing, k.s, k.attack.family) == (L.PIPE_BUCKET, 3, L.TAILOR_COORD)
    assert ops.pipeline_attack_job(x[5], x, 50, 50, [0, -1], [0], "clip", 0, "pipeline_uv", 1.0).mixing == L.PIPE_NONE
    for bad in (dict(attack="tailored_uv"), dict(rule="median"), dict(mixing="bucketing"), dict(mixing=("bucket", 0))):
        args = dict(rule="clip", attack="pipeline_uv", mixing=None)
        args.update(bad)
        with pytest.raises(L.RcmarlError):
            ops.pipeline_attack_job(x[5], x, 50, 50, [0, -1], [0], args["rule"], 0, args["attack"], 1.0,
                                    mixing=args["mixing"])


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


def trainer(mixing, aggregation, H=1, attack=("pipeline_std", 2.0)):
    from rcmarl.trainer import Trainer
    return Trainer(labels=BYZ, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing)


def built(excinfo):
    tb = excinfo.tb
    while tb is not None:
        if tb.tb_frame.f_code.co_name == "__init__" and "mixing" in tb.tb_frame.f_locals:
            return tb.tb_frame.f_locals["self"]
        tb = tb.tb_next
    raise AssertionError("no Trainer frame")


@pytest.mark.parametrize("mixing,aggregation", [
    (None, "dnc"), ("nnm", "krum"), ("bucket", "gmed"), ("nnm", "dnc"), (("bucket", 3), "clip"), ("bucket", "dnc"),
    (["nnm", ("bucket", 2), None, "bucket", None], ["krum", "clip", "mkrum", "dnc", "clip"]),
    (None, ["clip", "trim", "scclip", "wmsr", "clip"]),
])
def test_trainer_accepts_pipeline_attackers_for_every_rule_and_mixing(no_device, mixing, aggregation):
    for attack in (("pipeline_std", 2.0), ("pipeline_uv", 1.0), ("pipeline_sgn", 0.0)):
        with pytest.raises(no_device) as ex:
            trainer(mixing, aggregation, attack=attack)
        tr = built(ex)
        assert tr.pipe_pairs == [0, 1, 2] and tr.tailor_pairs == [] and tr.gamma_pairs == [0, 1, 2]


@pytest.mark.parametrize("mixing,aggregation", [(None, "dnc"), ("nnm", "clip"), ("bucket", "trim")])
def test_tailored_attack_stays_refused_where_it_was(no_device, mixing, aggregation):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="tailored attack does not model"):
        trainer(mixing, aggregation, attack=("tailored_std", 2.0))


def test_pipeline_pairs_follow_the_adaptive_and_tailored_pairs_in_gamma_pairs(no_device):
    from rcmarl.trainer import Trainer
    labels = ["Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative", "Byzantine", "Cooperative"]
    in_nodes = [[i, (i + 1) % 7, (i + 2) % 7, (i + 3) % 7] for i in range(7)]
    attack = [None, ("pipeline_uv", 1.0), None, ("minmax_std", 1.0), None, ("tailored_sgn", 2.0), None]
    with pytest.raises(no_device) as ex:
        Trainer(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((7, 2)), H=1, attack=attack)
    tr = built(ex)
    kind = {e: tr.attack[b][0] for e, (b, _, _) in enumerate(tr.byz_pairs)}
    assert tr.gamma_pairs == tr.adapt_pairs + tr.tailor_pairs + tr.pipe_pairs
    assert tr.pipe_pairs and all(isinstance(kind[e], type(kind[tr.pipe_pairs[0]])) for e in tr.pipe_pairs)
    assert {tr.byz_pairs[e][0] for e in tr.pipe_pairs} == {1}
