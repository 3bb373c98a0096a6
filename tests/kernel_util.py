"""Helpers shared by the kernel parity tests (test_kernels_gpu.py, test_kernel_shapes_gpu.py, test_minibatch_fit_gpu.py):
the library handle, the library's own CTA plan, seeded synthetic buffer rows, random networks, host -> device copies and
the tolerance check."""
import ctypes as C

import numpy as np
import pytest


def load_kernels():
    """The rcmarl bindings and cuda:0, or a skip when there is no CUDA device."""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from rcmarl import ops, nets, _lib
    _lib.lib()                                           # fail loudly if the .so is missing

    class NS:
        pass
    k = NS()
    k.ops, k.nets, k.L = ops, nets, _lib
    k.dev = torch.device("cuda:0")
    return k


def grad_ctas(K, NA, kinds, loss, n_rows, sms, balanced=False):
    """CTAs per job of a one-wave grid over n_rows rows on sms SMs, from the library's own plan: equal shares as
    rcmarl_grad launches them, or cost-balanced shares (balanced=True) as rcmarl_minibatch_fit launches its chains
    (n_rows = one mini-batch)."""
    n = len(kinds)
    out = (C.c_int32 * n)()
    K.L.check(K.L.lib().rcmarl_grad_grid_plan(NA, (C.c_int32 * n)(*kinds), n, loss, n_rows, int(balanced), sms, out),
              "rcmarl_grad_grid_plan")
    return list(out)


def synth(rs, B, NA=5, nrow=5):
    pos = rs.randint(0, nrow, size=(B, NA, 2))
    npos = np.clip(pos + rs.randint(-1, 2, size=pos.shape), 0, nrow - 1)
    mean, std = (nrow - 1) / 2.0, np.std(np.arange(nrow))
    s = ((pos - mean) / std).astype(np.float32)
    ns = ((npos - mean) / std).astype(np.float32)
    a = rs.randint(0, 5, size=(B, NA, 1)).astype(np.float32)
    r = (-rs.randint(0, 2 * nrow, size=(B, NA, 1)) / 5.0).astype(np.float32)
    return s, ns, a, r


def rand_net(rs, d_in, n_out):
    from rcmarl import nets
    w = nets.glorot_uniform(d_in, n_out, rs)
    return [x + (0.05 * rs.randn(*x.shape)).astype(np.float32) for x in w]


def to_dev(K, *arrs):
    import torch
    return [torch.as_tensor(np.ascontiguousarray(a)).to(K.dev) for a in arrs]


def close(got, want, rtol=1e-4, atol=1e-6, err_msg=""):
    if hasattr(got, "detach"):
        got = got.detach().cpu().numpy()
    got = np.asarray(got)
    np.testing.assert_allclose(got.astype(np.float64), np.asarray(want, np.float64), rtol=rtol, atol=atol,
                               err_msg=err_msg)
