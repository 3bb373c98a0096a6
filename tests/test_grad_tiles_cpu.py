"""Host view of the fit kernels' weight-gradient tiles (TileLayout, grad_kernel.cuh): every packed parameter of every
network the kernels fit is accumulated exactly once -- by one tile element or by the per-lane output-layer path of the
scalar nets -- and the phase-2 issue per buffer row is the one DESIGN.md 4.2 documents."""
import ctypes as C

import numpy as np
import pytest

NACT = 5
# (d_in, n_out): critic / actor at n_agents = 5, team reward at 5, and the 16-agent nets
LAYOUTS = [(10, 1), (15, 1), (32, 1), (48, 1), (10, NACT), (32, NACT)]
# warp-FFMA per buffer row in phase 2 (DESIGN.md 4.2); 32 everywhere with 8x8 tiles
PH2_PER_ROW = {(10, 1): 22, (15, 1): 28, (32, 1): 64, (48, 1): 64, (10, NACT): 64, (32, NACT): 64}


def tile_map(d_in, n_out):
    from rcmarl import _lib as L
    info = (C.c_int32 * 6)()
    cap = 32 * 64
    params = (C.c_int32 * cap)()
    L.check(L.lib().rcmarl_grad_tile_map(d_in, n_out, info, params, cap), "rcmarl_grad_tile_map")
    nt, ta, td, ng, ffma, first_out = list(info)
    return dict(nt=nt, ta=ta, td=td, ng=ng, ffma=ffma, first_out=first_out,
                params=np.array(params[:nt * ta * td]).reshape(nt, ta, td))


@pytest.mark.parametrize("d_in,n_out", LAYOUTS)
def test_every_parameter_is_accumulated_exactly_once(d_in, n_out):
    from rcmarl import _lib as L
    m = tile_map(d_in, n_out)
    n_params = L.param_count(d_in, n_out)
    assert m["nt"] * m["ng"] <= 32 and 64 % m["ng"] == 0
    assert m["ta"] * m["td"] <= 64                      # no more accumulators per lane than the 8x8 tile held
    p = m["params"].ravel()
    tiles = p[p >= 0]
    outside = np.arange(m["first_out"], n_params)        # per-lane W3 / b3 of the scalar nets (none for the actor)
    assert (n_out == 1) == (outside.size == 20 * n_out + n_out)
    seen = np.bincount(np.concatenate([tiles, outside]), minlength=n_params)
    assert seen.size == n_params and np.all(seen == 1), np.flatnonzero(seen != 1)


@pytest.mark.parametrize("d_in,n_out", LAYOUTS)
def test_phase2_issue_per_row(d_in, n_out):
    m = tile_map(d_in, n_out)
    assert m["ffma"] == (64 // m["ng"]) * m["ta"] * m["td"]
    assert m["ffma"] == 64 * PH2_PER_ROW[(d_in, n_out)]


def test_scalar_net_tiles_at_five_agents():
    """The n_agents = 5 critic and team-reward nets: padding is what is left of the per-row issue after the useful
    hidden-layer MACs (nets.n_hidden_params) are spread over all 32 lanes."""
    from rcmarl import nets
    crit, team = tile_map(10, 1), tile_map(15, 1)
    assert (crit["ta"], crit["td"], crit["nt"], crit["ng"]) == (11, 4, 15, 2)
    assert (team["ta"], team["td"], team["nt"], team["ng"]) == (8, 7, 15, 2)
    for m, din in ((crit, 10), (team, 15)):
        useful = int((m["params"] >= 0).sum())
        assert useful == nets.n_hidden_params(din)
        assert m["ffma"] // 64 * 32 >= useful


def test_unsupported_shapes_are_rejected():
    from rcmarl import _lib as L
    info = (C.c_int32 * 6)()
    params = (C.c_int32 * 4)()
    assert L.lib().rcmarl_grad_tile_map(11, 1, info, params, 4) == -1
    assert L.lib().rcmarl_grad_tile_map(10, 1, info, params, 4) == -1          # params too small for 15 tiles
