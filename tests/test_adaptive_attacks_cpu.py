"""CPU checks of the min-max / min-sum attacks (rcmarl_adaptive_attack, include/rcmarl.h): properties of the fp64 oracle
(tests/adaptive_attack_oracle.py) with hypothesis -- the message meets its constraint with equality, gamma >= 0, the
degenerate cases send mu, the honest list's order only matters through rounding, and the closed form is the limit of a
bisection of the constraint --, the hook against attack_oracle's for the older attacks, the C layout of the job, and the
refusals of the library, the bindings and Trainer before any device work."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import adaptive_attack_oracle as AA
import attack_oracle as AT
from test_attacks_cpu import _team5, no_device, trainer   # noqa: F401  (no_device is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f64 = np.float64
TIGHT = 1e-6


@st.composite
def honest_sets(draw, n_min=1):
    """n honest rows of P values on a grid of 1/16 (exact in fp64, so the degenerate cases are exact), repeats likely"""
    n = draw(st.integers(n_min, 16))
    P = draw(st.integers(1, 6))
    base = draw(st.lists(st.lists(st.integers(-800, 800), min_size=P, max_size=P), min_size=1, max_size=n))
    idx = draw(st.lists(st.integers(0, len(base) - 1), min_size=n, max_size=n))
    scale = draw(st.sampled_from([1.0, 1 / 16, 1e-3, 40.0]))
    return np.array([base[i] for i in idx], f64) * scale


@given(honest_sets(), st.sampled_from(AA.ATTACKS))
@settings(max_examples=400, deadline=None)
def test_the_message_meets_its_constraint_with_equality(v, attack):
    m, g = AA.craft(v, attack, 1.0)
    assert g >= 0 and np.isfinite(m).all()
    q, c = AA.constraint(v, attack, m)
    if g > 0:
        assert 1 - TIGHT <= q / c <= 1 + TIGHT, (q, c, g)
    else:
        np.testing.assert_array_equal(m, AT.moments(v)[0])


@given(honest_sets(), st.sampled_from(AA.ATTACKS), st.floats(0, 4))
@settings(max_examples=200, deadline=None)
def test_gamma_is_never_negative_and_does_not_depend_on_the_scale(v, attack, s):
    m, g = AA.craft(v, attack, s)
    g1 = AA.craft(v, attack, 1.0)[1]
    assert g >= 0 and g == g1
    mu, d, _ = AA.gamma_of(v, attack)
    np.testing.assert_allclose(m, mu + s * g * d, rtol=1e-12, atol=1e-12 * (1 + np.abs(mu).max() + s * g))


@given(st.lists(st.integers(-100, 100), min_size=1, max_size=6), st.integers(1, 16), st.sampled_from(AA.ATTACKS))
@settings(max_examples=100, deadline=None)
def test_degenerate_honest_sets_give_gamma_zero_and_the_mean(row, n, attack):
    for v in (np.array([row], f64), np.repeat(np.array([row], f64), n, 0)):   # n = 1; identical rows (c = 0)
        m, g = AA.craft(v, attack, 1.0)
        assert g == 0
        np.testing.assert_array_equal(m, AT.moments(v)[0])


@pytest.mark.parametrize("attack", AA.ATTACKS)
def test_a_zero_direction_gives_gamma_zero(attack):
    v = np.array([[1.0, -2.0, 0.5], [-1.0, 2.0, -0.5], [3.0, 0.0, 0.0], [-3.0, 0.0, 0.0]])   # mu = 0
    if attack.endswith("_std"):
        v = np.array([[1.0, -2.0, 0.5]] * 3)                                                  # sigma = 0
    mu, d, g = AA.gamma_of(v, attack)
    assert not d.any() and g == 0
    np.testing.assert_array_equal(AA.craft(v, attack, 2.0)[0], mu)


@given(honest_sets(n_min=2), st.sampled_from(AA.ATTACKS), st.randoms(use_true_random=False))
@settings(max_examples=200, deadline=None)
def test_permuting_the_honest_list_changes_gamma_only_by_rounding(v, attack, rnd):
    g = AA.craft(v, attack, 1.0)[1]
    perm = list(range(v.shape[0]))
    rnd.shuffle(perm)
    gp = AA.craft(v[perm], attack, 1.0)[1]
    np.testing.assert_allclose(gp, g, rtol=1e-9, atol=1e-12)


def _bisect(v, attack, steps=60):
    """the largest g >= 0 with the constraint met at mu + g d, by doubling then 60 halvings (the paper's search)"""
    mu, d, _ = AA.gamma_of(v, attack)

    def ok(g):
        q, c = AA.constraint(v, attack, mu + g * d)
        return q <= c
    if not ok(0.0):
        return 0.0
    hi = 1.0
    while ok(hi):
        hi *= 2
    lo = 0.0
    for _ in range(steps):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


@given(honest_sets(n_min=2), st.sampled_from(AA.ATTACKS))
@settings(max_examples=200, deadline=None)
def test_closed_form_is_the_limit_of_the_bisection(v, attack):
    mu, d, g = AA.gamma_of(v, attack)
    if not d.any():
        assert g == 0
        return
    b = _bisect(v, attack)
    np.testing.assert_allclose(g, b, rtol=1e-7, atol=1e-9 * (1 + b))


def test_fp32_oracle_is_close_to_fp64():
    rs = np.random.RandomState(41)
    for n in (2, 5, 16):
        v = (rs.randn(n, 761) * 0.3 + rs.randn(761)).astype(np.float32)
        for attack in AA.ATTACKS:
            m32, g32 = AA.craft(v, attack, 1.0)
            m64, g64 = AA.craft(v.astype(f64), attack, 1.0)
            assert g32.dtype == np.float32 and m32.dtype == np.float32
            np.testing.assert_allclose(g32, g64, rtol=1e-4)
            np.testing.assert_allclose(m32, m64, rtol=0, atol=1e-4 * np.abs(m64).max())


def test_hook_crafts_the_older_attacks_as_attack_oracle_does():
    labels = ["Cooperative"] * 4 + ["Byzantine"]
    ags, in_nodes, _ = _team5(labels)
    msgs, tmsgs = [ag.critic for ag in ags], [ag.TR for ag in ags]
    for attack in (("alie", 1.5), ("ipm", 0.5), ("gauss", 0.3)):
        want = AT.make_hook(labels, in_nodes, {4: attack}, seed=3, round_=7)(2, msgs, tmsgs)
        gam = {}
        got = AA.make_hook(labels, in_nodes, {4: attack}, seed=3, round_=7, gammas=gam)(2, msgs, tmsgs)
        assert gam == {}
        for x, y in zip(got, want):
            for j in range(4):
                for a, b in zip(x[j], y[j]):
                    for p, q in zip(a, b):
                        np.testing.assert_array_equal(p, q)
    gam = {}
    per_c, _ = AA.make_hook(labels, in_nodes, {4: ("minmax_std", 1.0)}, gammas=gam)(0, msgs, tmsgs)
    assert sorted(gam) == [(4, 1), (4, 2), (4, 3)] and all(len(g) == 2 and min(g) > 0 for g in gam.values())
    vals = np.stack([AT.pack(msgs[k], f64) for k in (1, 2, 3)])
    np.testing.assert_array_equal(AT.pack(per_c[1][3], f64), AA.craft(vals, "minmax_std", 1.0)[0])


# ------------------------------------------------------------------------------------------------ C ABI / bindings
def test_adaptive_attack_job_layout_as_gcc_sees_the_header(tmp_path):
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    fields = ["dst", "msgs", "msg_stride", "gamma_out", "n", "n_honest", "honest", "kind", "dev", "scale", "reserved"]
    enums = ["RCMARL_ADAPT_MINMAX", "RCMARL_ADAPT_MINSUM", "RCMARL_DEV_UV", "RCMARL_DEV_STD", "RCMARL_DEV_SGN",
             "RCMARL_ADAPTIVE_MAX_FLOATS"]
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rcmarl.h"\nint main(){'
                   'printf("%zu", sizeof(rcmarl_adaptive_attack_job));'
                   + "".join(f'printf(" %zu", offsetof(rcmarl_adaptive_attack_job, {f}));' for f in fields)
                   + "".join(f'printf(" %d", (int)({e}));' for e in enums) + 'printf("\\n"); return 0;}')
    exe = tmp_path / "off"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == ctypes.sizeof(L.AdaptiveAttackJob) == 120
    assert got[1:1 + len(fields)] == [getattr(L.AdaptiveAttackJob, f).offset for f in fields]
    assert got[1 + len(fields):] == [L.ADAPT_MINMAX, L.ADAPT_MINSUM, L.DEV_UV, L.DEV_STD, L.DEV_SGN,
                                     L.ADAPTIVE_MAX_FLOATS] == [0, 1, 0, 1, 2, 18 * 1536]
    assert ("rcmarl_adaptive_attack", ctypes.c_int, [ctypes.POINTER(L.AdaptiveAttackJob), ctypes.c_int, L.c_fp]) in L.SYMBOLS
    assert L.ADAPTIVE_ATTACKS == {f"{k}_{d}": (i, j) for i, k in enumerate(AA.KINDS) for j, d in enumerate(AA.DEVS)}


P_FAKE, STRIDE = 100, 128                       # fake device addresses: rows of msgs at 1 MiB + r * 512 bytes
MSGS = 1 << 20


def _job(**kw):
    from rcmarl import _lib as L
    j = L.AdaptiveAttackJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.n_honest = 1 << 24, MSGS, STRIDE, P_FAKE, 2
    j.kind, j.dev, j.scale = L.ADAPT_MINMAX, L.DEV_STD, 1.0
    j.honest[0], j.honest[1] = 0, 1
    for k, v in kw.items():
        if k == "honest":
            for i, x in enumerate(v):
                j.honest[i] = x
        else:
            setattr(j, k, v)
    return j


ROW5 = MSGS + 5 * STRIDE * 4


@pytest.mark.parametrize("bad", [
    dict(dst=None), dict(msgs=None), dict(n=0), dict(n=-3), dict(n_honest=0), dict(n_honest=17), dict(honest=[0, -1]),
    dict(kind=2), dict(kind=-1), dict(dev=3), dict(dev=-1), dict(scale=float("nan")), dict(scale=float("inf")),
    dict(scale=-0.5), dict(scale=float("-inf")),
    dict(n=18 * 1536 // 4 + 1, msg_stride=8192),                       # (2 + 2) * n over the staging bound
    dict(n=1537, n_honest=16, honest=list(range(16))),                 # (16 + 2) * n over the staging bound
    dict(dst=MSGS + STRIDE * 4 - 8),                                   # dst overlaps honest row 1 (of this job)
    dict(dst=ROW5 + 40, honest=[2, 3]),                                # ... an honest row of the other job
    dict(gamma_out=MSGS + 3 * STRIDE * 4 + 12, honest=[2, 3]),         # gamma_out on one of its honest rows
    dict(gamma_out=ROW5 + 4 * 8),                                      # ... on the other job's honest row
    dict(gamma_out=(1 << 25) + 4),                                     # ... on the other job's dst
    dict(gamma_out=1 << 26),                                           # ... on the other job's gamma_out
    dict(dst=(1 << 25) + 4 * (P_FAKE - 1)),                            # two dsts overlap
])
def test_library_refuses_bad_jobs_without_a_device(bad):
    from rcmarl import _lib as L
    lib = L.lib()
    good = _job(dst=1 << 25, gamma_out=1 << 26, honest=[5, 6])
    for jobs in ([good, _job(**bad)], [_job(**bad), good]):
        arr = (L.AdaptiveAttackJob * len(jobs))(*jobs)
        assert lib.rcmarl_adaptive_attack(arr, len(arr), None) == -1           # RCMARL_ERR_ARG


def test_staging_bound_is_the_trainers_largest_job():
    from rcmarl import _lib as L
    assert (16 + 2) * L.param_count(48, 1) <= L.ADAPTIVE_MAX_FLOATS < (16 + 2) * 1537
    assert 4 * L.ADAPTIVE_MAX_FLOATS + 1168 <= 227 * 1024          # with the kernel's static shared memory, per CTA


def test_library_refuses_bad_job_counts_without_a_device():
    from rcmarl import _lib as L
    lib = L.lib()
    assert lib.rcmarl_adaptive_attack(None, 1, None) == -1
    arr = (L.AdaptiveAttackJob * 33)(*[_job(dst=(1 << 24) + (1 << 12) * i) for i in range(33)])
    assert lib.rcmarl_adaptive_attack(arr, 0, None) == -1
    assert lib.rcmarl_adaptive_attack(arr, 33, None) == -1


def test_attack_names_and_parameters():
    from rcmarl import _lib as L
    for name in AA.ATTACKS:
        kind, s = L.check_attack((name, 1))
        assert kind == L.ADAPTIVE_ATTACKS[name] and isinstance(kind, tuple) and s == 1.0
        assert L.check_attack((name, 0)) == (kind, 0.0) and L.is_adaptive_attack(name)
        for bad in [(name, -1e-3), (name, float("nan")), (name, float("inf")), (name, "x"), (name,)]:
            with pytest.raises(L.RcmarlError):
                L.check_attack(bad)
    assert L.check_attack(("alie", -2)) == (0, -2.0)                  # the older attacks keep their ids
    for bad in [("minmax", 1), ("minsum_l2", 1), ("MINMAX_UV", 1), ((0, 1), 1.0)]:
        with pytest.raises(L.RcmarlError):
            L.check_attack(bad)
    assert not L.is_adaptive_attack("alie") and not L.is_adaptive_attack((0, 0))


def test_bindings_refuse_unknown_names():
    import torch
    from rcmarl import _lib as L, ops
    x = torch.zeros(4, 8)
    with pytest.raises(L.RcmarlError):
        ops.adaptive_attack_job(x[3], x, 8, 8, [0, 1], "minmax", 1.0)
    with pytest.raises(L.RcmarlError):
        ops.adaptive_attack_job(x[3], x, 8, 8, [0, 1], "alie", 1.0)
    j = ops.adaptive_attack_job(x[3], x, 8, 8, [0, 1, 2], "minsum_sgn", 0.5, gamma_out=x[3, :1])
    assert (j.kind, j.dev, j.n_honest, j.scale, j.gamma_out) == (1, 2, 3, 0.5, x[3].data_ptr())


@pytest.mark.parametrize("attack", [("minmax_std", -1.0), ("minsum_uv", float("nan")), ("minmax", 1.0),
                                    [None] * 4 + [("minsum_sgn", float("inf"))]])
def test_trainer_refuses_invalid_adaptive_attacks_before_any_device_work(no_device, attack):   # noqa: F811
    from rcmarl import _lib as L
    with pytest.raises(L.RcmarlError):
        trainer(attack, H=0)


@pytest.mark.parametrize("attack,labels", [
    (("minmax_std", 1.0), None),
    ([None] * 4 + [("minsum_uv", 0.0)], None),
    ([("minmax_sgn", 2.0), None, ("alie", 1.0), None, None], ["Byzantine", "Cooperative", "Byzantine", "Cooperative",
                                                            "Cooperative"]),
])
def test_trainer_accepts_adaptive_attacks(no_device, attack, labels):   # noqa: F811
    with pytest.raises(no_device):
        trainer(attack, labels)
