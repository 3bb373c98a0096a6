"""CPU checks of the ARC-aware Byzantine messages (rcmarl_pipeline_arc_attack, rcmarl_history_arc_attack,
include/rcmarl.h): the symbols as gcc sees the header and the bindings declare them, the library's refusals without a
device (one float past each staging bound included), the attack names, the Trainer's refusals and acceptances before it
touches a device, every field of the ARC jobs it builds, and the oracle (tests/arc_attack_oracle.py): at H = 0 ARC is
the identity and the ARC craft is the pipeline / history craft."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import arc_attack_oracle as AAO
import history_attack_oracle as HO
import pipeline_attack_oracle as PA
import test_history_attack_cpu as HC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
SLOTS, HONEST = HC.SLOTS, HC.HONEST
no_device, built, C5, BYZ = HC.no_device, HC.built, HC.C5, HC.BYZ


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("rule", PA.RULES)
@pytest.mark.parametrize("mixing", [None, "nnm", ("bucket", 2)])
def test_at_h0_the_pipeline_form_is_the_pipeline_oracle(rule, mixing):
    rs = np.random.RandomState(13100 + len(rule))
    X = HC._stack(rs, dtype=np.float64)
    for d in ("uv", "std", "sgn"):
        m, g, O, R, c = AAO.craft_pipeline(X, SLOTS, HONEST, rule, 0, "arc_" + d, 2.0, mixing=mixing, n_perms=2)
        pm, pg, pO, pR = PA.craft(X, SLOTS, HONEST, rule, 0, "pipeline_" + d, 2.0, mixing=mixing, n_perms=2)
        assert np.array_equal(m, pm) and g == pg and np.array_equal(O, pO) and np.array_equal(R, pR)
        assert (c == 1).all()


@pytest.mark.parametrize("rule", PA.RULES)
@pytest.mark.parametrize("dtype", [np.float64, f32])
def test_at_h0_the_history_form_is_the_history_oracle(rule, dtype):
    rs = np.random.RandomState(13200 + len(rule))
    X = HC._stack(rs, dtype=dtype)
    c = (X[0] + rs.randn(X.shape[1]) * 0.1).astype(dtype)
    M = (rs.randn(len(SLOTS), X.shape[1]) * 0.2).astype(dtype)
    for d in ("uv", "std", "sgn"):
        m, g, O, R, f = AAO.craft_history(X, SLOTS, HONEST, rule, 0, "arc_" + d, 2.0, c, M, 0.9, False, [1, 4])
        hm, hg, hO, hR, _ = HO.craft(X, SLOTS, HONEST, rule, 0, "history_" + d, 2.0, c, M, 0.9, False, [1, 4])
        assert np.array_equal(m, hm) and g == hg and np.array_equal(O, hO) and np.array_equal(R, hR)
        assert (f == 1).all()


def test_at_h_one_the_modelled_aggregate_is_the_rule_of_the_clipped_rows():
    """H = 1 at n_in = 8 (k_clip = 1): R(gamma_i*) is the rule over arc_oracle.clip of the slots with the message."""
    rs = np.random.RandomState(13300)
    X = HC._stack(rs, dtype=np.float64)
    for rule in ("clip", "mkrum", "dnc"):
        m, g, O, R, c = AAO.craft_pipeline(X, SLOTS, HONEST, rule, 1, "arc_std", 2.0)
        Y = AAO.AO.clip(np.stack([m if s < 0 else X[s] for s in SLOTS]), 1)[0]
        assert np.array_equal(R, PA.rule_output(Y, rule, 1)) and c.shape == (2,)
    with pytest.raises(ValueError):
        AAO.craft_pipeline(X, [-1] + SLOTS[1:], HONEST[1:], "clip", 1, "arc_std", 2.0)     # a crafted slot 0


# ------------------------------------------------------------------------------------------------ C ABI
def test_symbols_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "arc.c"
    src.write_text('#include "rcmarl.h"\nint main(){'
                   'int (*p)(const rcmarl_pipeline_attack_job*, int, void*) = rcmarl_pipeline_arc_attack;'
                   'int (*h)(const rcmarl_history_attack_job*, int, void*) = rcmarl_history_arc_attack;'
                   'return (p(0, 0, 0) | h(0, 0, 0)) ? 1 : 0;}')
    stub = tmp_path / "stub.c"
    stub.write_text('#include "rcmarl.h"\n'
                    'int rcmarl_pipeline_arc_attack(const rcmarl_pipeline_attack_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}\n'
                    'int rcmarl_history_arc_attack(const rcmarl_history_attack_job* j, int n, void* s)'
                    '{(void)j; (void)n; (void)s; return 0;}')
    exe = tmp_path / "arc"
    subprocess.check_call(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), str(stub), "-o", str(exe)])
    subprocess.check_call([str(exe)])
    lib = L.lib()
    assert lib.rcmarl_pipeline_arc_attack.argtypes == [ctypes.POINTER(L.PipelineAttackJob), ctypes.c_int, L.c_fp]
    assert lib.rcmarl_history_arc_attack.argtypes == [ctypes.POINTER(L.HistoryAttackJob), ctypes.c_int, L.c_fp]
    assert lib.rcmarl_pipeline_arc_attack.restype == lib.rcmarl_history_arc_attack.restype == ctypes.c_int


def _pjob(mixing=0, **kw):
    """A valid pipeline job on made-up addresses (the history test's C2 receiver), with `mixing`."""
    from rcmarl import _lib as L
    h = HC._job(**kw)
    j = L.PipelineAttackJob()
    j.attack, j.model_out, j.mixing = h.attack, h.model_out, mixing
    j.s, j.n_perms = 2, 2
    return j


@pytest.mark.parametrize("bad", HC.BAD[:22] + HC.BAD[-7:-3] + [dict(slots=[-1, 1, 2, 3], honest_mask=0b1010)])
def test_pipeline_form_refuses_what_the_base_refuses_and_a_crafted_slot_0(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    other = _pjob(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000)
    for jobs in ([_pjob(**bad)], [other, _pjob(**bad)]):
        arr = (L.PipelineAttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_pipeline_arc_attack(arr, len(arr), None) == -1, bad


@pytest.mark.parametrize("bad", HC.BAD + [dict(slots=[-1, 1, 2, 3], honest_mask=0b1010, own_mask=0b0001)])
def test_history_form_refuses_what_the_base_refuses_and_a_crafted_slot_0(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    other = HC._job(dst=1 << 26, gamma_out=(1 << 26) + 4 * 8000, model_out=(1 << 26) + 4 * 9000)
    for jobs in ([HC._job(**bad)], [other, HC._job(**bad)]):
        arr = (L.HistoryAttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_history_arc_attack(arr, len(arr), None) == -1, bad


def test_one_float_past_each_staging_bound_is_refused_without_a_device():
    """The bound holds the base staging plus k_clip * n floats: n_in = 16 with 15 real slots at H = 1 (k_clip = 1).
    History: (16 + 4 + 1) * n <= 22 * 1421 admits n = 1488 and refuses 1489.  Pipeline under nnm: (15 + 16 + 4 + 1) *
    n <= 37 * 1421 admits n = 1460 and refuses 1461, which the base attacks' bounds admit.  Only refused jobs are
    passed to the library: an admitted job on made-up addresses would launch."""
    from rcmarl import _lib as L
    lib = L.lib()
    common = dict(n_in=16, slots=list(range(15)) + [-1], honest_mask=(1 << 15) - 1, H=1, msg_stride=2000,
                  dst=1 << 28, gamma_out=1 << 27, model_out=(1 << 27) + 64)
    assert (16 + 4 + 1) * 1488 <= L.HISTORY_MAX_FLOATS < (16 + 4 + 1) * 1489
    assert (15 + 16 + 4 + 1) * 1460 <= L.PIPELINE_MAX_FLOATS < (15 + 16 + 4 + 1) * 1461
    assert (16 + 4) * 1489 <= L.HISTORY_MAX_FLOATS and (15 + 16 + 4) * 1461 <= L.PIPELINE_MAX_FLOATS
    j = HC._job(n=1489, momentum_stride=2000, own_mask=1 << 15, **common)
    assert lib.rcmarl_history_arc_attack((L.HistoryAttackJob * 1)(j), 1, None) == -1
    j = _pjob(mixing=L.PIPE_NNM, n=1461, **common)
    assert lib.rcmarl_pipeline_arc_attack((L.PipelineAttackJob * 1)(j), 1, None) == -1


def test_refuses_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_pipeline_arc_attack(None, 1, None) == -1 and lib.rcmarl_history_arc_attack(None, 1, None) == -1
    arr = (L.HistoryAttackJob * 33)(*[HC._job(dst=(1 << 26) + 4 * 1000 * i, gamma_out=(1 << 27) + 4 * i,
                                              model_out=(1 << 28) + 4 * 1000 * i) for i in range(33)])
    assert lib.rcmarl_history_arc_attack(arr, 0, None) == -1 and lib.rcmarl_history_arc_attack(arr, 33, None) == -1


def test_attack_names_and_bindings():
    import torch
    from rcmarl import _lib as L, ops
    assert sorted(L.ARC_ATTACKS) == ["arc_sgn", "arc_std", "arc_uv"]
    for d, dev in (("uv", 0), ("std", 1), ("sgn", 2)):
        kind, param = L.check_attack((f"arc_{d}", 2))
        assert isinstance(kind, L.ArcAttackKind) and int(kind) == dev and param == 2.0
        assert not isinstance(kind, (L.HistoryKind, L.PipelineKind, L.TailoredKind))
        assert L.is_arc_attack(f"arc_{d}") and not L.is_history_attack(f"arc_{d}")
    assert L.check_attack(("arc_std", 0.0))[1] == 0.0
    for bad in (("arc_uv", -0.5), ("arc_std", float("nan")), ("arc_sgn", float("inf")), ("arc", 1.0), ("arc_dnc", 1.0)):
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)
    x = torch.zeros(8, 50)
    M = torch.zeros(4, 60)
    j = ops.history_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "clip", 1, "arc_sgn", 1.5, x[6], M, 60, 0.9,
                               1, [2])
    assert j.attack.dev == L.DEV_SGN and j.attack.scale == 1.5
    j = ops.pipeline_attack_job(x[5], x, 50, 50, [0, 1, -1, 3], [0, 1, 3], "dnc", 1, "arc_uv", 1.0, mixing="nnm")
    assert (j.attack.dev, j.attack.family, j.mixing) == (L.DEV_UV, L.TAILOR_SPECTRAL, L.PIPE_NNM)
    assert callable(ops.pipeline_arc_attack) and callable(ops.history_arc_attack)


# ------------------------------------------------------------------------------------------------ Trainer
def trainer(aggregation, momentum=None, clipping="arc", attack=("arc_std", 2.0), mixing=None, H=1, **kw):
    from rcmarl.trainer import Trainer
    return Trainer(labels=BYZ, in_nodes=C5, weights=[], desired=np.zeros((5, 2)), H=H, aggregation=aggregation,
                   attack=attack, mixing=mixing, momentum=momentum, clipping=clipping, **kw)


@pytest.mark.parametrize("aggregation,momentum,mixing,clipping", [
    ("clip", None, None, "arc"), ("dnc", 0.9, None, "arc"), ("mkrum", None, "nnm", "arc"),
    ("gmed", None, ("bucket", 2), "arc"), ("trim", None, None, None), ("scclip", 0.9, None, None),
    (["krum", "trim", "scclip", "dnc", "clip"], [None, 0.9, None, None, None], [None, None, "nnm", None, None],
     ["arc", "arc", None, "arc", None]),
])
def test_trainer_accepts_arc_attackers(no_device, aggregation, momentum, mixing, clipping):
    for attack in (("arc_std", 2.0), ("arc_uv", 1.0), ("arc_sgn", 0.0)):
        with pytest.raises(no_device) as ex:
            trainer(aggregation, momentum, clipping, attack=attack, mixing=mixing)
        tr = built(ex)
        assert tr.arc_pairs == [0, 1, 2] and tr.hist_pairs == tr.pipe_pairs == [] and tr.gamma_pairs == [0, 1, 2]


@pytest.mark.parametrize("rule", ["mda", "smea"])
@pytest.mark.parametrize("clipping", [None, "arc"])
def test_trainer_refuses_arc_attacks_against_subset_rules(no_device, rule, clipping):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match=f"ARC attack against agent .*'{rule}' the attack does not model"):
        trainer(rule, clipping=clipping)


@pytest.mark.parametrize("name", ["tailored_std", "pipeline_uv", "history_sgn"])
def test_older_adaptive_attacks_stay_refused_against_clipping(no_device, name):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="whose clipping 'arc' the attack does not model"):
        trainer("clip", attack=(name, 2.0))


def test_trainer_refuses_a_job_past_the_staging_bound(no_device):
    """16 agents in one clique of 16 under nnm at H = 2 (k_clip = 3): (15 + 16 + 4 + 3) * 1421 > 37 * 1421."""
    from rcmarl import _lib as L
    from rcmarl.trainer import Trainer
    labels = ["Cooperative"] * 15 + ["Byzantine"]
    in_nodes = [[i] + [k for k in range(16) if k != i] for i in range(16)]
    kw = dict(labels=labels, in_nodes=in_nodes, weights=[], desired=np.zeros((16, 2)), aggregation="clip",
              mixing="nnm", clipping="arc", attack=[None] * 15 + [("arc_std", 2.0)])
    with pytest.raises(L.RcmarlError, match="more than the 52577 the library admits"):
        Trainer(H=2, **kw)
    with pytest.raises(no_device):                      # H = 1: k_clip = 1, 36 rows
        Trainer(H=1, **kw)


@pytest.mark.parametrize("s", [-1.0, float("nan"), float("inf")])
def test_trainer_refuses_a_bad_scale(no_device, s):
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError, match="needs a finite parameter"):
        trainer("clip", attack=("arc_uv", s))


def _cpu_trainer(monkeypatch, **kw):
    import torch
    from rcmarl import ops
    from rcmarl.trainer import Trainer
    monkeypatch.setattr(ops, "workspace", lambda *a, **k: torch.zeros(8, dtype=torch.uint8))
    return Trainer(weights=[], H=1, device="cpu", **kw)


def _check_base(tr, j, e, t, r, slots, honest_mask, dev, scale, rule=None):
    from rcmarl import _lib as L
    NA = tr.NA
    msgs, P = (tr.msg_c, tr.PC) if t == 0 else (tr.msg_t, tr.PT)
    a = j.attack
    assert (a.dst, a.msgs, a.msg_stride, a.n, a.n_in) == (msgs[NA + e].data_ptr(), msgs.data_ptr(), P, P, len(slots))
    assert list(a.slots[:a.n_in]) == slots and a.honest_mask == honest_mask
    assert (a.family, a.rule) == (rule or (L.TAILOR_COORD, L.AGG_CLIP)) and (a.H, a.dev, a.scale) == (1, dev, scale)
    assert a.gamma_out == tr.att_gamma[tr.gamma_pairs.index(e), t:t + 1].data_ptr() and j.model_out is None


def test_job_layout_with_momentum_mixing_bucketing_and_plain_receivers(monkeypatch):
    """Attackers 4 and 5 (receiver 2 lists 4 twice) against receiver 0 (clips alone), 1 (clips before nnm), 2 (momentum
    then clipping), 3 (clips before bucketing) and 6 (does not clip, momentum): every field of every job, the launch
    each group goes to, and the momentum index of each history-form job."""
    from rcmarl import _lib as L, ops
    labels = ["Cooperative"] * 4 + ["Byzantine"] * 2 + ["Cooperative"]
    in_nodes = [[0, 1, 4, 3], [1, 2, 4, 5], [2, 4, 3, 4, 5], [3, 0, 5, 1], [4, 0, 1, 2], [5, 0, 1, 2], [6, 5, 0, 1]]
    mom = [None, None, 0.9, None, None, None, 0.5]
    mixing = [None, "nnm", None, ("bucket", 2), None, None, None]
    clip = ["arc", "arc", "arc", "arc", None, None, None]
    tr = _cpu_trainer(monkeypatch, labels=labels, in_nodes=in_nodes, desired=np.zeros((7, 2)), momentum=mom,
                      mixing=mixing, clipping=clip, attack=[None] * 4 + [("arc_std", 2.0), ("arc_uv", 1.0), None])
    assert tr.byz_pairs == [(4, 0, [0, 1, 3]), (4, 1, [1, 2]), (4, 2, [2, 3]), (5, 1, [1, 2]), (5, 2, [2, 3]),
                            (5, 3, [3, 0, 1]), (5, 6, [6, 0, 1])]
    assert tr.arc_pairs == list(range(7)) and tr.gamma_pairs == tr.arc_pairs and tr.mom_agents == [2, 6]
    assert all(g == [] for g in tr._attack_job_groups())    # the ARC pairs get no other job
    groups = tr._arc_job_groups()
    assert [(g[0], len(g[1]), g[2]) for g in groups] == [
        (ops.history_arc_attack, 4, [0, 0, 0, 0]), (ops.history_attack, 2, [1, 1]),
        (ops.pipeline_arc_attack, 8, None)]
    hist_arc, hist_plain, pipe_arc = (list(g[1]) for g in groups)
    for n, (e, t) in enumerate((e, t) for e in (2, 4) for t in (0, 1)):
        j = hist_arc[n]
        dev, scale = (L.DEV_STD, 2.0) if e == 2 else (L.DEV_UV, 1.0)
        _check_base(tr, j, e, t, 2, [2, -1, 3, -1, -1], 0b00101, dev, scale)
        ref = tr.critic[2] if t == 0 else tr.tr[2]
        assert (j.ref, j.momentum, j.momentum_stride) == (ref.data_ptr(), tr.momentum_M[0, t].data_ptr(), tr.PT)
        assert j.beta == f32(0.9) and j.first == 0 and j.own_mask == (0b01010 if e == 2 else 0b10000)
    for n, t in enumerate((0, 1)):
        j = hist_plain[n]
        _check_base(tr, j, 6, t, 6, [6, -1, 0, 1], 0b1101, L.DEV_UV, 1.0)
        assert j.momentum == tr.momentum_M[1, t].data_ptr() and j.beta == f32(0.5) and j.own_mask == 0b0010
    want = {0: (0, [0, 1, -1, 3], 0b1011, None), 1: (1, [1, 2, -1, -1], 0b0011, "nnm"),
            3: (1, [1, 2, -1, -1], 0b0011, "nnm"), 5: (3, [3, 0, -1, 1], 0b1011, ("bucket", 2))}
    for j, (e, t) in zip(pipe_arc, ((e, t) for e in (0, 1, 3, 5) for t in (0, 1))):
        r, slots, hm, mix = want[e]
        dev, scale = (L.DEV_STD, 2.0) if tr.byz_pairs[e][0] == 4 else (L.DEV_UV, 1.0)
        _check_base(tr, j, e, t, r, slots, hm, dev, scale)
        assert j.mixing == (L.PIPE_NONE if mix is None else L.PIPE_NNM if mix == "nnm" else L.PIPE_BUCKET)
        assert j.s == (2 if mix == ("bucket", 2) else 0) and j.n_perms == L.PIPELINE_PERMS
        assert (j.seed, j.attacker, j.receiver, j.net, j.round) == (tr.seed, tr.byz_pairs[e][0], r, t, 0)


def test_a_receiver_that_does_not_clip_gets_the_history_attacks_jobs(monkeypatch):
    """Without clipping anywhere, the ARC pairs' jobs are field for field those of the same history attack, and they
    go to rcmarl_history_attack / rcmarl_pipeline_attack."""
    from rcmarl import ops
    labels = ["Cooperative"] * 4 + ["Byzantine"] * 2
    in_nodes = [[0, 1, 2, 3], [1, 2, 4, 5], [2, 4, 3, 4, 5], [3, 0, 5, 1], [4, 0, 1, 2], [5, 0, 1, 2]]
    mom = [0.9, None, 0.99, 0.5, None, None]
    kw = dict(labels=labels, in_nodes=in_nodes, desired=np.zeros((6, 2)), momentum=mom)
    arc = _cpu_trainer(monkeypatch, attack=[None] * 4 + [("arc_std", 2.0), ("arc_uv", 1.0)], **kw)
    hist = _cpu_trainer(monkeypatch, attack=[None] * 4 + [("history_std", 2.0), ("history_uv", 1.0)], **kw)
    groups = arc._arc_job_groups()
    assert [g[0] for g in groups] == [ops.history_attack, ops.pipeline_attack]
    _, _, _, pipe, hg, hist_mom, _, _, _ = hist._attack_job_groups()
    assert groups[0][2] == hist_mom

    def fields(j, tr):
        out = []
        for name, _ in type(j)._fields_:
            v = getattr(j, name)
            if name == "attack":
                v = [(n, list(getattr(v, n)) if n == "slots" else getattr(v, n)) for n, _ in type(v)._fields_]
            out.append((name, v))
        return out
    for (_, ga, _), gb in ((groups[0], hg[0][1]), (groups[1], pipe[0])):
        assert len(ga) == len(gb)
        for ja, jb in zip(ga, gb):
            fa, fb = fields(ja, arc), fields(jb, hist)
            for (na, va), (nb, vb) in zip(fa, fb):
                if na == "attack":                    # pointers into each trainer's own buffers
                    va = [(n, x) for n, x in va if n not in ("dst", "msgs", "gamma_out")]
                    vb = [(n, x) for n, x in vb if n not in ("dst", "msgs", "gamma_out")]
                elif na in ("ref", "momentum"):
                    continue
                assert va == vb, na


def test_an_attacker_listed_twice_owns_both_slots(monkeypatch):
    from rcmarl import ops
    labels = ["Cooperative"] * 4 + ["Byzantine"]
    in_nodes = [[0, 4, 1, 4], [1, 2, 3, 0], [2, 3, 0, 1], [3, 0, 1, 2], [4, 0, 1, 2]]
    for mom, launch in ((0.9, ops.history_arc_attack), (None, ops.pipeline_arc_attack)):
        tr = _cpu_trainer(monkeypatch, labels=labels, in_nodes=in_nodes, desired=np.zeros((5, 2)), momentum=mom,
                          clipping="arc", attack=[None] * 4 + [("arc_sgn", 1.0)])
        assert tr.arc_pairs == [0]
        (fn, g, _), = tr._arc_job_groups()
        assert fn == launch and len(g) == 2
        for j in g:
            assert list(j.attack.slots[:4]) == [0, -1, 1, -1] and j.attack.honest_mask == 0b0101
            if mom is not None:
                assert j.own_mask == 0b1010


def test_without_an_arc_attacker_no_arc_groups(monkeypatch):
    labels = ["Cooperative"] * 4 + ["Byzantine"]
    tr = _cpu_trainer(monkeypatch, labels=labels, in_nodes=C5, desired=np.zeros((5, 2)), clipping="arc",
                      attack=[None] * 4 + [("gauss", 1.0)])
    assert tr.arc_pairs == [] and tr._arc_job_groups() == []
