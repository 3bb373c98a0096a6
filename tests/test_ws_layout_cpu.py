"""Host-side check of the 3xTF32 split arithmetic (tools/experiments/tf32x3_error.py); no GPU.  No shipped kernel uses this
split: the test guards only the tensor-core fit design of DESIGN.md §7, for a future kernel built on it."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_tf32x3_split_error_stays_at_fp32_level():
    """3xTF32 with a truncating split of the activations (the form the design uses) against fp64: within 4e-7 of max|z| for the two
    layer shapes of the nets, without bias (tools/experiments/tf32x3_error.py restates the kernel's arithmetic in NumPy)."""
    t = _load(os.path.join(ROOT, "tools", "experiments", "tf32x3_error.py"), "tf32x3_error")
    rs = np.random.RandomState(1)
    for K in (16, 24):
        A = rs.uniform(-2, 2, (512, K)).astype(np.float32)
        lim = np.sqrt(6.0 / (K + 20))
        B = rs.uniform(-lim, lim, (K, 20)).astype(np.float32)
        ref = A.astype(np.float64) @ B.astype(np.float64)
        b_hi = t.tf32_rna(B)
        b_lo = t.tf32_trunc(B - b_hi)
        a_hi = t.tf32_trunc(A)
        a_lo = t.tf32_trunc(A - a_hi)
        x = t.mm32(a_hi, b_hi) + t.mm32(a_lo, b_hi) + t.mm32(a_hi, b_lo)
        scale = np.abs(ref).max()
        assert np.abs(x - ref).max() / scale < 4e-7
        assert abs((x - ref).mean()) / scale < 2e-8
        one_pass = t.mm32(t.tf32_trunc(A), t.tf32_trunc(B))
        assert np.abs(one_pass - ref).max() / scale > 1e-4          # what the split buys
