"""NumPy emulation of the 3xTF32 split of the tensor-core fit design in DESIGN.md §7, which no shipped kernel uses (A_hi.B_hi + A_lo.B_hi + A_hi.B_lo; weights B: hi = value
rounded to tf32 with round-to-nearest-away; activations A: hi either rounded (three ops per element) or TRUNCATED to tf32 (two
ops, the measured form); lo = value - hi, truncated to tf32 by the tensor core; fp32 accumulation): error of one hidden layer of
the RPBCAC nets against fp64, max and mean signed (bias), next to plain fp32 and single-pass TF32.  CPU only.
    python tools/experiments/tf32x3_error.py
"""
import numpy as np


def tf32_rna(x):
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x1000) & 0xFFFFE000            # cvt.rna.tf32.f32: add half an ulp of the 10-bit mantissa, drop 13 bits
    return u.astype(np.uint32).view(np.float32)


def tf32_trunc(x):
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def mm32(a, b):
    """fp32 accumulation in k order (the tensor core's internal order is not specified; this is the pessimistic case)."""
    out = np.zeros((a.shape[0], b.shape[1]), np.float32)
    for k in range(a.shape[1]):
        out += a[:, k:k + 1].astype(np.float32) * b[k:k + 1, :].astype(np.float32)
    return out


def main():
    rs = np.random.RandomState(0)
    for name, K in (("layer 1 (x | 1) . [W1; b1], K = 16", 16), ("layer 2 (h1 | 1) . [W2; b2], K = 24", 24)):
        A = rs.uniform(-2, 2, (4096, K)).astype(np.float32)
        lim = np.sqrt(6.0 / (K + 20))
        B = rs.uniform(-lim, lim, (K, 20)).astype(np.float32)
        ref = A.astype(np.float64) @ B.astype(np.float64)
        scale = np.abs(ref).max()
        a_hi, b_hi = tf32_rna(A), tf32_rna(B)
        a_lo, b_lo = tf32_trunc(A - a_hi), tf32_trunc(B - b_hi)
        x3 = mm32(a_hi, b_hi) + mm32(a_lo, b_hi) + mm32(a_hi, b_lo)
        t_hi = tf32_trunc(A)
        t_lo = tf32_trunc(A - t_hi)
        x3t = mm32(t_hi, b_hi) + mm32(t_lo, b_hi) + mm32(t_hi, b_lo)
        x1 = mm32(tf32_trunc(A), tf32_trunc(B))
        f32 = mm32(A, B)
        print(f"{name}: max |err| / max |z|   fp32 FMA order {np.abs(f32 - ref).max() / scale:.2e}   "
              f"3xTF32 {np.abs(x3 - ref).max() / scale:.2e}   3xTF32 truncating A split {np.abs(x3t - ref).max() / scale:.2e}   "
              f"1xTF32 {np.abs(x1 - ref).max() / scale:.2e}")
        print(f"    mean signed error / max |z| (bias)   fp32 {(f32 - ref).mean() / scale:+.1e}   3xTF32 {(x3 - ref).mean() / scale:+.1e}   "
              f"truncating {(x3t - ref).mean() / scale:+.1e}")


if __name__ == "__main__":
    main()
