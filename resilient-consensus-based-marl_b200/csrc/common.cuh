// common.cuh -- shared device helpers for the RPBCAC sm_90a kernels.
// Network layout and math follow main.py:60-82 (Dense 20 / LeakyReLU(0.1)), see include/rcmarl.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "rcmarl.h"

namespace rcmarl {

constexpr int HID = RCMARL_HIDDEN;
constexpr int NACT = RCMARL_N_ACTIONS;
constexpr float SLOPE = 0.1f;

// last CUDA error of the calling thread (rcmarl_last_cuda_error); defined in train_kernels.cu
int last_cuda_error_get();
void last_cuda_error_set(int e);
#define RC_CUDA(x)                                              \
    do {                                                        \
        cudaError_t e_ = (x);                                   \
        if (e_ != cudaSuccess) {                                \
            rcmarl::last_cuda_error_set((int)e_);               \
            return RCMARL_ERR_CUDA;                             \
        }                                                       \
    } while (0)

__host__ __device__ constexpr int param_count(int din, int nout) {
    return din * HID + HID + HID * HID + HID + HID * nout + nout;
}
__host__ __device__ constexpr int off_b1(int din) { return din * HID; }
__host__ __device__ constexpr int off_W2(int din) { return din * HID + HID; }
__host__ __device__ constexpr int off_b2(int din) { return din * HID + HID + HID * HID; }
__host__ __device__ constexpr int off_W3(int din) { return din * HID + 2 * HID + HID * HID; }
__host__ __device__ constexpr int off_b3(int din, int nout) { return off_W3(din) + HID * nout; }
__host__ __device__ constexpr int round4(int n) { return (n + 3) & ~3; }

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may start
// its prologue while its predecessor drains; it must not touch the predecessor's outputs before pdl_wait().
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ float lrelu(float z) { return z > 0.f ? z : SLOPE * z; }
// derivative expressed through the activation output (sign(h) == sign(z), slope > 0);
// tf.nn.leaky_relu passes alpha*g at z == 0
__device__ __forceinline__ float lrelu_grad_from_out(float h) { return h > 0.f ? 1.f : SLOPE; }

// absolute buffer row of the m-th processed row (rcmarl_rows, include/rcmarl.h)
__device__ __forceinline__ int64_t row_of(const rcmarl_rows& R, int64_t m) {
    if (R.time_idx == nullptr) return R.row_begin + m;
    int64_t q = m / R.n_envs;
    return R.row_begin + (int64_t)R.time_idx[q] * R.n_envs + (m - q * R.n_envs);
}

// Network input of one buffer row, Keras Flatten order (train_agents.py:89-93).
//   IN_SA: sa[row][0:3NA]      IN_NS: ns[row][0:2NA]      IN_S: sa[row] without the action column
template <int NA, int DIN>
__device__ __forceinline__ void load_x(const rcmarl_rows& R, int kind, int64_t row, float (&x)[DIN]) {
    if (DIN == 3 * NA) {
        const float* p = R.sa + row * (3 * NA);
#pragma unroll
        for (int k = 0; k < DIN; ++k) x[k] = __ldg(p + k);
    } else {
        const bool is_ns = (kind == RCMARL_IN_NS);
        const float* p = is_ns ? (R.ns + row * (2 * NA)) : (R.sa + row * (3 * NA));
        const int sel = is_ns ? 0 : 1;
#pragma unroll
        for (int k = 0; k < DIN; ++k) x[k] = __ldg(p + k + sel * (k >> 1));
    }
}

// cooperative global -> shared copy of one packed network (n floats, n % 4 == 0 not required)
__device__ __forceinline__ void stage_weights(float* dst, const float* __restrict__ src, int n) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = __ldg(src + i);
}

// z = b + x W  (W row-major [K][20] in shared memory, broadcast float4 reads), then LeakyReLU
template <int K>
__device__ __forceinline__ void dense20(const float* __restrict__ sW, const float* __restrict__ sb,
                                        const float (&x)[K], float (&h)[HID]) {
#pragma unroll
    for (int q = 0; q < HID / 4; ++q) {
        float4 v = reinterpret_cast<const float4*>(sb)[q];
        h[4 * q + 0] = v.x; h[4 * q + 1] = v.y; h[4 * q + 2] = v.z; h[4 * q + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float4* w = reinterpret_cast<const float4*>(sW + k * HID);
#pragma unroll
        for (int q = 0; q < HID / 4; ++q) {
            float4 v = w[q];
            h[4 * q + 0] = fmaf(x[k], v.x, h[4 * q + 0]);
            h[4 * q + 1] = fmaf(x[k], v.y, h[4 * q + 1]);
            h[4 * q + 2] = fmaf(x[k], v.z, h[4 * q + 2]);
            h[4 * q + 3] = fmaf(x[k], v.w, h[4 * q + 3]);
        }
    }
#pragma unroll
    for (int j = 0; j < HID; ++j) h[j] = lrelu(h[j]);
}

// features of one row: h2 = lrelu(lrelu(x W1 + b1) W2 + b2)   (critic_features / TR_features,
// agents/resilient_CAC_agents.py:39-40)
template <int DIN>
__device__ __forceinline__ void features(const float* __restrict__ sw, const float (&x)[DIN],
                                         float (&h1)[HID], float (&h2)[HID]) {
    dense20<DIN>(sw, sw + off_b1(DIN), x, h1);
    dense20<HID>(sw + off_W2(DIN), sw + off_b2(DIN), h1, h2);
}

template <int DIN>
__device__ __forceinline__ float head1(const float* __restrict__ sw, const float (&h2)[HID]) {
    const float* W3 = sw + off_W3(DIN);
    float out = sw[off_b3(DIN, 1)];
#pragma unroll
    for (int j = 0; j < HID; ++j) out = fmaf(h2[j], W3[j], out);
    return out;
}

template <int DIN>
__device__ __forceinline__ void head5(const float* __restrict__ sw, const float (&h2)[HID],
                                      float (&logit)[NACT]) {
    const float* W3 = sw + off_W3(DIN);
    const float* b3 = sw + off_b3(DIN, NACT);
#pragma unroll
    for (int o = 0; o < NACT; ++o) logit[o] = b3[o];
#pragma unroll
    for (int j = 0; j < HID; ++j)
#pragma unroll
        for (int o = 0; o < NACT; ++o) logit[o] = fmaf(h2[j], W3[j * NACT + o], logit[o]);
}

// softmax in place; returns log-sum-exp pieces for the cross-entropy
__device__ __forceinline__ void softmax5(float (&l)[NACT], float& mx, float& lse) {
    mx = l[0];
#pragma unroll
    for (int o = 1; o < NACT; ++o) mx = fmaxf(mx, l[o]);
    float s = 0.f;
#pragma unroll
    for (int o = 0; o < NACT; ++o) { l[o] = expf(l[o] - mx); s += l[o]; }
    lse = logf(s);
    const float inv = 1.f / s;
#pragma unroll
    for (int o = 0; o < NACT; ++o) l[o] *= inv;
}

// Coordinate-wise clipped mean of n values, own = v[0]
// (RPBCAC_agent._resilient_aggregation, agents/resilient_CAC_agents.py:42-58).
// Order statistics by rank counting: n <= 16, exact for ties.
template <int MAXN>
__device__ __forceinline__ float clip_mean_small(const float (&v)[MAXN], int n, int H) {
    float sH = v[0], sT = v[0];
    const int rT = n - H - 1;
#pragma unroll
    for (int k = 0; k < MAXN; ++k) {
        if (k < n) {
            int rank = 0;
#pragma unroll
            for (int m = 0; m < MAXN; ++m)
                if (m < n) rank += (v[m] < v[k] || (v[m] == v[k] && m < k)) ? 1 : 0;
            if (rank == H) sH = v[k];
            if (rank == rT) sT = v[k];
        }
    }
    const float lo = fminf(sH, v[0]);
    const float hi = fmaxf(sT, v[0]);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < MAXN; ++k)
        if (k < n) s += fmaxf(fminf(v[k], hi), lo);
    return s / (float)n;
}

// Resilient aggregation of n values under rule (rcmarl_agg_rule, include/rcmarl.h), own = v[0].  CLIP is
// clip_mean_small; TRIM and WMSR keep the ranks lo..hi of the same tie-broken rank count and add the kept values in
// index order, so that a dropped outlier (1e30, +-inf) never touches the sum.  The branch is uniform per job.
template <int MAXN>
__device__ __forceinline__ float resilient_mean_small(const float (&v)[MAXN], int n, int H, int rule) {
    if (rule == RCMARL_AGG_CLIP) return clip_mean_small<MAXN>(v, n, H);
    int lo = H, hi = n - H - 1;
    if (rule == RCMARL_AGG_WMSR) {            // at most H strictly above own and at most H strictly below it
        int above = 0, below = 0;
#pragma unroll
        for (int k = 1; k < MAXN; ++k) {
            if (k < n) {
                above += v[k] > v[0] ? 1 : 0;
                below += v[k] < v[0] ? 1 : 0;
            }
        }
        lo = min(H, below);
        hi = n - 1 - min(H, above);
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < MAXN; ++k) {
        if (k < n) {
            int rank = 0;
#pragma unroll
            for (int m = 0; m < MAXN; ++m)
                if (m < n) rank += (v[m] < v[k] || (v[m] == v[k] && m < k)) ? 1 : 0;
            if (rank >= lo && rank <= hi) s += v[k];
        }
    }
    return s / (float)(hi - lo + 1);
}

// A pair of fp32 values (two adjacent hidden units, or two accumulators) updated together.  Hopper has no packed fp32
// FMA, so a pair operation is two IEEE fp32 FMAs (FFMA); the values are the same as one packed operation would give.
typedef float2 f2;
__device__ __forceinline__ f2 pack2(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ void unpack2(f2 v, float& lo, float& hi) {
    lo = v.x;
    hi = v.y;
}
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// LeakyReLU of a packed pair.  slope in (0, 1) => lrelu(z) == max(z, slope * z) bit for bit (z > 0: slope*z < z;
// z < 0: slope*z > z; +-0 and NaN map to themselves), which is 2 x (FMUL, FMNMX) instead of 2 x (FMUL, FSETP, FSEL).
__device__ __forceinline__ void lrelu_pair(f2 z, float& a, float& b) {
    float za, zb, ta, tb;
    unpack2(z, za, zb);
    unpack2(mul2(z, pack2(SLOPE, SLOPE)), ta, tb);
    a = fmaxf(za, ta);
    b = fmaxf(zb, tb);
}

// z[r][:] = b + x[r] W for R rows at once (W row-major [K][20] and b [20] in shared memory, broadcast float4 reads):
// every weight quad feeds 4*R FFMA; outputs are packed as pairs of adjacent hidden units.
template <int K, int R>
__device__ __forceinline__ void dense20_rows(const float* __restrict__ sW, const float* __restrict__ sb,
                                             const float (&x)[R][K], float (&h)[R][HID]) {
    f2 hp[R][HID / 2];
#pragma unroll
    for (int q = 0; q < HID / 4; ++q) {
        const float4 v = reinterpret_cast<const float4*>(sb)[q];
#pragma unroll
        for (int r = 0; r < R; ++r) { hp[r][2 * q] = pack2(v.x, v.y); hp[r][2 * q + 1] = pack2(v.z, v.w); }
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
        f2 xk[R];
#pragma unroll
        for (int r = 0; r < R; ++r) xk[r] = pack2(x[r][k], x[r][k]);
        const float4* w = reinterpret_cast<const float4*>(sW + k * HID);
#pragma unroll
        for (int q = 0; q < HID / 4; ++q) {
            const float4 v = w[q];
            const f2 w0 = pack2(v.x, v.y), w1 = pack2(v.z, v.w);
#pragma unroll
            for (int r = 0; r < R; ++r) {
                hp[r][2 * q] = fma2(xk[r], w0, hp[r][2 * q]);
                hp[r][2 * q + 1] = fma2(xk[r], w1, hp[r][2 * q + 1]);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int j = 0; j < HID / 2; ++j) lrelu_pair(hp[r][j], h[r][2 * j], h[r][2 * j + 1]);
}

// hidden features of R rows at once (critic_features / TR_features, agents/resilient_CAC_agents.py:39-40)
template <int DIN, int R>
__device__ __forceinline__ void features_rows(const float* __restrict__ sw, const float (&x)[R][DIN],
                                              float (&h1)[R][HID], float (&h2)[R][HID]) {
    dense20_rows<DIN, R>(sw, sw + off_b1(DIN), x, h1);
    dense20_rows<HID, R>(sw + off_W2(DIN), sw + off_b2(DIN), h1, h2);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace rcmarl
