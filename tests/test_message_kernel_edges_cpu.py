"""The fp64 oracles of the whole-message kernels (vector_oracle, dnc_oracle, nnm_oracle, bucket_oracle,
adaptive_attack_oracle, tailored_attack_oracle, pipeline_attack_oracle, dissensus_mimic_oracle) against the closed forms
of tests/edge_inputs.py: identical messages (G = 0 for DnC), two clusters, rows on a line, repeated in-nodes, one
parameter, and squared distances that overflow or underflow in fp32.  Each oracle runs on the fp32 messages (the
kernels' inputs) and on the same values in fp64; selections and weights must equal the closed form exactly, outputs
bitwise in fp32 and in fp64 up to the one rounding of the fp32 division.  No GPU and no library."""
import numpy as np
import pytest

import adaptive_attack_oracle as AA
import bucket_oracle as BO
import dissensus_mimic_oracle as DM
import dnc_oracle as DO
import edge_inputs as E
import nnm_oracle as NO
import pipeline_attack_oracle as PA
import tailored_attack_oracle as TA
import vector_oracle as VO

CASES = E.edge_cases()
IDS = [c.name for c in CASES]
DTYPES = (np.float32, np.float64)


def _same(got, want, dt, tag):
    if dt == np.float32:
        np.testing.assert_array_equal(np.asarray(got, np.float32), want, err_msg=tag)
    else:
        np.testing.assert_allclose(np.asarray(got, np.float64), want.astype(np.float64), rtol=2.0 ** -23,
                                   atol=2.0 ** -23 * float(np.abs(want.astype(np.float64)).max(initial=0.0)), err_msg=tag)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("rule", ["krum", "mkrum"])
def test_krum_oracle_matches_the_closed_form(case, rule, dt):
    w, out = E.krum(case, rule)
    got, gw = VO.aggregate(case.X.astype(dt), case.H, rule)
    np.testing.assert_array_equal(gw > 0, w > 0, err_msg=f"{case} {rule}")
    _same(got, out, dt, f"{case} {rule}")


SCCLIP = [c for c in CASES if c.P == 1 or c.name.split("_")[0] in ("identical", "overflow", "underflow")]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", SCCLIP, ids=[c.name for c in SCCLIP])
def test_scclip_oracle_matches_the_closed_form(case, dt):
    if case.name.startswith("two_clusters"):
        pytest.skip("d_k is not exact")
    w, out = E.scclip(case)
    got, gw = VO.aggregate(case.X.astype(dt), case.H, "scclip")
    _same(gw, w, dt, str(case))
    _same(got, out, dt, str(case))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("P", E.EDGE_P)
def test_gmed_oracle_at_the_magnitude_edges(P, dt):
    """Overflow: only the median row is at a finite distance, out = that row.  Identical rows and underflow: every
    distance is 0, every beta_k is 1 / nu, the weights are equal."""
    case = E.scaled(P, E.OVER, "overflow")
    w, out = E.gmed_overflow(case)
    got, gw = VO.aggregate(case.X.astype(dt), case.H, "gmed")
    _same(gw, w, dt, str(case))
    _same(got, out, dt, str(case))
    for case in (E.identical(P), E.scaled(P, E.UNDER, "underflow")):
        got, gw = VO.aggregate(case.X.astype(dt), case.H, "gmed")
        if dt == np.float32 or case.name.startswith("identical"):
            assert (gw == gw[0]).all(), f"{case}: {gw}"
        if case.name.startswith("identical"):
            _same(got, case.X[0], dt, str(case))


@pytest.mark.parametrize("dt", DTYPES)
def test_gmed_oracle_stays_on_the_line(dt):
    case = E.collinear()
    got, _ = VO.aggregate(case.X.astype(dt), case.H, "gmed")
    c, v = case.X[0].astype(np.float64), (case.X[1].astype(np.float64) - case.X[0]) / 3
    s = float((got - c) @ v / (v @ v))
    np.testing.assert_allclose(got, c + s * v, rtol=0, atol=1e-5 * np.abs(case.X).max())
    assert min(case.t) < s < max(case.t)


DNC = [c for c in CASES if c.t is not None]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", DNC, ids=[c.name for c in DNC])
def test_dnc_oracle_matches_the_closed_form(case, dt):
    """Rows on a line: DnC removes the H largest |t_k - mean t| (at scale 2^64 and 2^-84 too: fp64 centring); identical
    rows (G = 0, every eigenvector equally valid): every score is 0 and the H highest indices go."""
    assert DO.removed(case.X.astype(dt), case.H) == E.dnc_removed(case), str(case)
    w, out = E.dnc(case)
    got, gw = DO.aggregate(case.X.astype(dt), case.H)
    np.testing.assert_array_equal(gw > 0, w > 0, err_msg=str(case))
    _same(got, out, dt, str(case))


@pytest.mark.parametrize("H", range(0, 7))
@pytest.mark.parametrize("P", E.EDGE_P)
def test_dnc_oracle_on_identical_rows_removes_the_highest_indices(P, H):
    case = E.identical(P, H=H)
    assert DO.removed(case.X, H) == list(range(7 - H, 7))
    assert (DO.scores(case.X) == 0).all()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_nnm_oracle_matches_the_closed_form(case, dt):
    sel, mixed = E.nnm(case)
    assert NO.selections(case.X.astype(dt), case.H) == sel, str(case)
    got, M = NO.mix(case.X.astype(dt), case.H)
    _same(got, mixed, dt, str(case))


@pytest.mark.parametrize("P", E.EDGE_P)
def test_bucket_oracle_on_identical_rows(P):
    case = E.identical(P)
    for s in (1, 2, 3, 6):
        got, M = BO.bucket_mix(case.X, s, 99, 3, 1, 7, 2)
        assert got.shape[0] == BO.n_out(case.n, s)
        np.testing.assert_array_equal(got, np.tile(case.X[0], (got.shape[0], 1)))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("values", [[3, -1, 7, 5, 1], [-6, 2, -4, 0, -2, -8, 4]])
def test_adaptive_oracle_sgn_at_one_parameter(values, dt):
    V = np.array(values, dt)[:, None]
    g, m = E.minmax_sgn_p1(values)
    msg, gg = AA.craft(V, "minmax_sgn", 1.0)
    assert gg == g and msg[0] == m, (gg, g, msg, m)
    g32, g_exact, m32 = E.minsum_sgn_p1(values)
    msg, gg = AA.craft(V, "minsum_sgn", 1.0)
    if dt == np.float32:
        assert gg == g32 and msg[0] == m32, (gg, g32, msg, m32)
    else:
        np.testing.assert_allclose(gg, g_exact, rtol=1e-12)


MU_CASES = [c for c in CASES if c.name.split("_")[0] in ("identical", "overflow", "underflow")]


@pytest.mark.parametrize("case", MU_CASES, ids=[c.name for c in MU_CASES])
def test_attack_oracles_send_the_mean_at_the_edges(case):
    """Identical rows, overflowing and underflowing distances: gamma = 0 for min-max / min-sum, and i* = 0, gamma = 0
    for the tailored and pipeline searches; the message is mu, the fp32 mean of the honest rows."""
    X = case.X
    mu = E.f32_mean(X[:5])
    for attack in AA.ATTACKS:
        msg, g = AA.craft(X[:5], attack, 1.0)
        assert g == 0 and np.array_equal(msg, mu), f"{case} {attack}"
    slots, honest = [0, 1, -1, 2, 3, -1, 4], [0, 1, 3, 4, 6]
    for rule in ("clip", "krum", "gmed"):
        msg, g, O = TA.craft(X, slots, honest, rule, 1, "tailored_sgn", 2.0)
        assert g == 0 and np.array_equal(msg, mu), f"{case} {rule}"
    for rule, mixing in (("dnc", None), ("mkrum", "nnm"), ("trim", ("bucket", 2))):
        msg, g, Ob, R = PA.craft(X, slots, honest, rule, 1, "pipeline_uv", 2.0, mixing=mixing, n_perms=2)
        assert g == 0 and np.array_equal(msg, mu), f"{case} {rule} {mixing}"


MIMIC = [c for c in CASES if c.t is not None]


@pytest.mark.parametrize("case", MIMIC, ids=[c.name for c in MIMIC])
def test_mimic_oracle_matches_the_closed_form(case):
    for cand in (list(range(case.n)), list(range(1, case.n, 2)), [k for k in range(case.n) if k != 6]):
        k, live = E.mimic(case, cand)
        got, z, t = DM.mimic(case.X, cand, np.zeros(case.P, np.float32), 0)
        assert got == k and bool(z.any()) == live, f"{case} {cand}: {got} {k}"


@pytest.mark.parametrize("case", [E.line(), E.identical(33), E.scaled(1421, E.OVER, "overflow")], ids=lambda c: c.name)
@pytest.mark.parametrize("n_byz,eps", [(1, 1.0), (2, 1.0), (4, 3.0), (2, 0.0)])
def test_dissensus_oracle_matches_the_closed_form(case, n_byz, eps):
    got = DM.dissensus(case.X[0], case.X, n_byz, eps)
    np.testing.assert_array_equal(got, E.dissensus(case, n_byz, eps))
    if eps == 0 or case.name.startswith("identical"):
        np.testing.assert_array_equal(got, case.X[0])
