// rollout_consensus.cu
//   clip_mean_kernel   K4 / C5: streaming coordinate-wise clipped mean over the neighbour axis
//                      (HBM-bound: one coalesced 16-byte read per lane per neighbour row,
//                      order statistics kept in registers, no sort, no second pass)
//   rollout_kernel     K1 + K8: episodes under a fixed policy, one thread per (episode, env)
//   env_step_kernel    Grid_World.step/get_data for the per-call API
// Reference: agents/resilient_CAC_agents.py:42-58,208-219; environments/grid_world.py:37-72;
// training/train_agents.py:46-80.
#include "common.cuh"

namespace rcmarl {

int sm_count_cached();

// ============================================================================================
// clip mean (SURVEY 3.4 single-pass identity):
//   sum_k clip(v_k, lo, hi) = sum_k v_k - sum_{small_k < lo}(small_k - lo) - sum_{large_k > hi}(large_k - hi)
// where small / large are the H+1 smallest / largest values, lo = min(s[H], own), hi = max(s[n-H-1], own).
// ============================================================================================
__device__ __forceinline__ float4 ld_stream(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

template <int H>
struct Track {
    float small[H + 1];  // ascending: small[H] is the (H+1)-th smallest
    float large[H + 1];  // descending: large[H] is the (H+1)-th largest
    float sum;
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int i = 0; i <= H; ++i) { small[i] = INFINITY; large[i] = -INFINITY; }
        sum = 0.f;
    }
    // Branch-free insertion: with 4 columns per lane and 32 lanes, "some column needs an insert" is true for
    // practically every row, so a threshold test only adds divergence.  2(2H+1) FMNMX + 1 FADD per element.
    __device__ __forceinline__ void push(float v) {
        sum += v;
        float c = v;
#pragma unroll
        for (int i = 0; i < H; ++i) { const float lo = fminf(small[i], c); c = fmaxf(small[i], c); small[i] = lo; }
        small[H] = fminf(small[H], c);
        c = v;
#pragma unroll
        for (int i = 0; i < H; ++i) { const float hi = fmaxf(large[i], c); c = fminf(large[i], c); large[i] = hi; }
        large[H] = fmaxf(large[H], c);
    }
    // Two values at once for H == 1: sort the pair, then the two smallest of {small[0] <= small[1], lo <= hi} are
    // min(small[0], lo) and min3(small[1], hi, max(small[0], lo)); likewise the two largest.  10 min / max per pair instead
    // of 12, same values and the same summation order as two push() calls.
    __device__ __forceinline__ void push2(float a, float b) {
        static_assert(H == 1, "pair update is written for H == 1");
        sum += a;
        sum += b;
        const float lo = fminf(a, b), hi = fmaxf(a, b);
        const float m = fmaxf(small[0], lo);
        small[0] = fminf(small[0], lo);
        small[1] = fminf(fminf(small[1], hi), m);
        const float w = fminf(large[0], hi);
        large[0] = fmaxf(large[0], hi);
        large[1] = fmaxf(fmaxf(large[1], lo), w);
    }
    __device__ __forceinline__ void window(float own, float& lo, float& hi) const {
        lo = fminf(small[H], own);
        hi = fmaxf(large[H], own);
    }
    // The single-pass identity subtracts the excess of the extremes from a running sum that CONTAINS them: exact in real
    // arithmetic, but in fp32 one huge (adversarial) value absorbs the honest ones before it cancels (0.1 + 1e8 - 1e8 = 0),
    // and an infinity gives inf - inf.  The identity is therefore only used while the most extreme value stays within
    // 16x of the clipping window (error <= 16 n eps of the window, the order of the reference's own fp32 mean); otherwise the
    // caller re-reads the column and sums clip(v, lo, hi) directly (second pass, taken for outlier columns only).
    __device__ __forceinline__ bool identity_ok(float lo, float hi) const {
        const float w = fmaxf(fabsf(lo), fabsf(hi));
        const float m = fmaxf(fabsf(small[0]), fabsf(large[0]));
        return m <= 16.f * w;                 // false for NaN / inf extremes and for w == 0 < m
    }
    __device__ __forceinline__ float finish(float lo, float hi, int n) const {
        float s = sum;
#pragma unroll
        for (int i = 0; i <= H; ++i) {
            s -= fminf(small[i] - lo, 0.f);   // values below lo are raised to lo
            s -= fmaxf(large[i] - hi, 0.f);   // values above hi are lowered to hi
        }
        return s / (float)n;
    }
};
// tf.clip_by_value(x, lo, hi) = max(min(x, hi), lo)   (agents/resilient_CAC_agents.py:55)
__device__ __forceinline__ float clip1(float v, float lo, float hi) { return fmaxf(fminf(v, hi), lo); }

// ---- sorting networks (optimal comparator counts, verified with the 0-1 principle in tools/gen_sortnets.py) ----
template <bool ASC>
__device__ __forceinline__ void cswap(float& a, float& b) {
    const float lo = fminf(a, b), hi = fmaxf(a, b);
    a = ASC ? lo : hi;
    b = ASC ? hi : lo;
}
template <int N> struct SortNet;
template <> struct SortNet<1> { template <bool ASC> static __device__ __forceinline__ void run(float (&)[1]) {} };
template <> struct SortNet<2> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[2]) { cswap<ASC>(a[0], a[1]); } };
template <> struct SortNet<3> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[3]) { cswap<ASC>(a[0], a[1]); cswap<ASC>(a[1], a[2]); cswap<ASC>(a[0], a[1]); } };
template <> struct SortNet<4> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[4]) { cswap<ASC>(a[0], a[1]); cswap<ASC>(a[2], a[3]); cswap<ASC>(a[0], a[2]); cswap<ASC>(a[1], a[3]); cswap<ASC>(a[1], a[2]); } };
template <> struct SortNet<5> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[5]) { cswap<ASC>(a[0], a[1]); cswap<ASC>(a[3], a[4]); cswap<ASC>(a[2], a[4]); cswap<ASC>(a[2], a[3]); cswap<ASC>(a[1], a[4]); cswap<ASC>(a[0], a[3]); cswap<ASC>(a[0], a[2]); cswap<ASC>(a[1], a[3]); cswap<ASC>(a[1], a[2]); } };
template <> struct SortNet<6> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[6]) { cswap<ASC>(a[1], a[2]); cswap<ASC>(a[4], a[5]); cswap<ASC>(a[0], a[2]); cswap<ASC>(a[3], a[5]); cswap<ASC>(a[0], a[1]); cswap<ASC>(a[3], a[4]); cswap<ASC>(a[2], a[5]); cswap<ASC>(a[0], a[3]); cswap<ASC>(a[1], a[4]); cswap<ASC>(a[2], a[4]); cswap<ASC>(a[1], a[3]); cswap<ASC>(a[2], a[3]); } };
template <> struct SortNet<7> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[7]) { cswap<ASC>(a[1], a[2]); cswap<ASC>(a[3], a[4]); cswap<ASC>(a[5], a[6]); cswap<ASC>(a[0], a[2]); cswap<ASC>(a[3], a[5]); cswap<ASC>(a[4], a[6]); cswap<ASC>(a[0], a[1]); cswap<ASC>(a[4], a[5]); cswap<ASC>(a[2], a[6]); cswap<ASC>(a[0], a[4]); cswap<ASC>(a[1], a[5]); cswap<ASC>(a[0], a[3]); cswap<ASC>(a[2], a[5]); cswap<ASC>(a[1], a[3]); cswap<ASC>(a[2], a[4]); cswap<ASC>(a[2], a[3]); } };
template <> struct SortNet<8> { template <bool ASC> static __device__ __forceinline__ void run(float (&a)[8]) { cswap<ASC>(a[0], a[2]); cswap<ASC>(a[1], a[3]); cswap<ASC>(a[4], a[6]); cswap<ASC>(a[5], a[7]); cswap<ASC>(a[0], a[4]); cswap<ASC>(a[1], a[5]); cswap<ASC>(a[2], a[6]); cswap<ASC>(a[3], a[7]); cswap<ASC>(a[0], a[1]); cswap<ASC>(a[2], a[3]); cswap<ASC>(a[4], a[5]); cswap<ASC>(a[6], a[7]); cswap<ASC>(a[2], a[4]); cswap<ASC>(a[3], a[5]); cswap<ASC>(a[1], a[4]); cswap<ASC>(a[3], a[6]); cswap<ASC>(a[1], a[2]); cswap<ASC>(a[3], a[4]); cswap<ASC>(a[5], a[6]); } };

// Group update for H >= 2: the 8 new values of a column are sorted once (19 comparators); the H+1 smallest of
// {kept smallest (ascending), sorted group} are the element-wise minima against the reversed group head (bitonic
// half-cleaner), re-sorted with a (H+1)-input network; same for the largest.  ~11 FMNMX per element for H = 4
// instead of 4H+2 for one-at-a-time insertion.
template <int H>
__device__ __forceinline__ void push_group8(Track<H>& t, float (&g)[8]) {
    constexpr int K = H + 1;
#pragma unroll
    for (int i = 0; i < 8; ++i) t.sum += g[i];
    SortNet<8>::run<true>(g);
#pragma unroll
    for (int i = 0; i < K; ++i) t.small[i] = fminf(t.small[i], g[K - 1 - i]);
    SortNet<K>::template run<true>(t.small);
#pragma unroll
    for (int i = 0; i < K; ++i) t.large[i] = fmaxf(t.large[i], g[8 - K + i]);
    SortNet<K>::template run<false>(t.large);
}

constexpr int CM_UNROLL = 8;

// VEC consecutive columns of one neighbour row as one streaming load (16 or 8 bytes per lane, read-only path, no L1 fill)
template <int VEC>
__device__ __forceinline__ void ld_stream_vec(const float* p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 r = ld_stream(reinterpret_cast<const float4*>(p));
        v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = r.w;
    } else {
        static_assert(VEC == 2, "vector width");
        asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(v[0]), "=f"(v[1]) : "l"(p));
    }
}

// One thread owns VEC adjacent columns.  VEC = 4 (16-byte loads) for H <= 1, where a column costs a handful of registers;
// VEC = 2 for H >= 2: the per-column state (2 (H + 1) order statistics + the 8-row group being sorted) is what limits
// occupancy there (round 1: 98 registers, 22 % occupancy, DRAM 55 % busy with the ALUs 45 % busy -- neither saturated, the
// loads of a thread's next row group simply were not in flight while it sorted the current one), and half the columns per
// thread doubles the resident warps that cover each other's load latency.  8-byte loads still fill whole 32-byte sectors.
template <int H, int VEC>
__global__ void __launch_bounds__(256) clip_mean_vec_kernel(const float* __restrict__ vals, int n, int64_t PV,
                                                            int64_t row_stride, float* __restrict__ out) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // vector column
    if (c >= PV) return;
    Track<H> t[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) t[q].init();
    const float* base = vals + c * VEC;
    float own[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) own[q] = 0.f;
    int k = 0;
    for (; k + CM_UNROLL <= n; k += CM_UNROLL) {
        float v[CM_UNROLL][VEC];
#pragma unroll
        for (int u = 0; u < CM_UNROLL; ++u) ld_stream_vec<VEC>(base + (int64_t)(k + u) * row_stride, v[u]);
        if (k == 0) {
#pragma unroll
            for (int q = 0; q < VEC; ++q) own[q] = v[0][q];
        }
        if constexpr (H >= 2) {
#pragma unroll
            for (int q = 0; q < VEC; ++q) {
                float g[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) g[u] = v[u][q];
                push_group8<H>(t[q], g);
            }
        } else if constexpr (H == 1) {
#pragma unroll
            for (int u = 0; u < CM_UNROLL; u += 2)
#pragma unroll
                for (int q = 0; q < VEC; ++q) t[q].push2(v[u][q], v[u + 1][q]);
        } else {
#pragma unroll
            for (int u = 0; u < CM_UNROLL; ++u)
#pragma unroll
                for (int q = 0; q < VEC; ++q) t[q].push(v[u][q]);
        }
    }
    for (; k < n; ++k) {
        float v[VEC];
        ld_stream_vec<VEC>(base + (int64_t)k * row_stride, v);
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
            if (k == 0) own[q] = v[q];
            t[q].push(v[q]);
        }
    }
    float lo[VEC], hi[VEC], r[VEC];
    bool ok = true;
#pragma unroll
    for (int q = 0; q < VEC; ++q) {
        t[q].window(own[q], lo[q], hi[q]);
        ok = ok && t[q].identity_ok(lo[q], hi[q]);
    }
    if (ok) {
#pragma unroll
        for (int q = 0; q < VEC; ++q) r[q] = t[q].finish(lo[q], hi[q], n);
    } else {                                   // outlier column(s): second pass, clip first, then sum (reference order)
#pragma unroll
        for (int q = 0; q < VEC; ++q) r[q] = 0.f;
        for (int kk = 0; kk < n; ++kk) {
            float v[VEC];
            ld_stream_vec<VEC>(base + (int64_t)kk * row_stride, v);
#pragma unroll
            for (int q = 0; q < VEC; ++q) r[q] += clip1(v[q], lo[q], hi[q]);
        }
#pragma unroll
        for (int q = 0; q < VEC; ++q) r[q] = r[q] / (float)n;
    }
    if constexpr (VEC == 4) reinterpret_cast<float4*>(out)[c] = make_float4(r[0], r[1], r[2], r[3]);
    else reinterpret_cast<float2*>(out)[c] = make_float2(r[0], r[1]);
}

template <int H>
__global__ void __launch_bounds__(256) clip_mean_scalar_kernel(const float* __restrict__ vals, int n, int64_t P,
                                                               int64_t row_stride, float* __restrict__ out) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= P) return;
    Track<H> t;
    t.init();
    float own = 0.f;
    for (int k = 0; k < n; ++k) {
        float v = __ldg(vals + (int64_t)k * row_stride + c);
        if (k == 0) own = v;
        t.push(v);
    }
    float lo, hi;
    t.window(own, lo, hi);
    if (t.identity_ok(lo, hi)) {
        out[c] = t.finish(lo, hi, n);
    } else {
        float sum = 0.f;
        for (int k = 0; k < n; ++k) sum += clip1(__ldg(vals + (int64_t)k * row_stride + c), lo, hi);
        out[c] = sum / (float)n;
    }
}

template <int H>
static int launch_clip_mean(const float* vals, int n, int64_t P, int64_t row_stride, float* out, cudaStream_t st) {
    constexpr int VEC = H >= 2 ? 2 : 4;
    const bool vec = (P % VEC == 0) && (row_stride % VEC == 0) && ((uintptr_t)vals % (4 * VEC) == 0) && ((uintptr_t)out % (4 * VEC) == 0);
    if (vec) {
        const int64_t PV = P / VEC;
        clip_mean_vec_kernel<H, VEC><<<(unsigned)((PV + 255) / 256), 256, 0, st>>>(vals, n, PV, row_stride, out);
    } else {
        clip_mean_scalar_kernel<H><<<(unsigned)((P + 255) / 256), 256, 0, st>>>(vals, n, P, row_stride, out);
    }
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

// ============================================================================================
// environment + rollout
// ============================================================================================
// grid_world.py:27 actions_dict: 0 stay, 1 (-1,0), 2 (+1,0), 3 (0,-1), 4 (0,+1)
__device__ __forceinline__ void move_of(int a, int& dx, int& dy) {
    dx = (a == 1) ? -1 : (a == 2 ? 1 : 0);
    dy = (a == 3) ? -1 : (a == 4 ? 1 : 0);
}
// One agent's transition + reward (grid_world.py:51-64).  The collision test at :56 includes the agent
// itself, so dist_to_agents == 0 always: reward = 0 if (on goal and action == 0) else -(pre-move distance) - 1.
// Both coordinates are clipped with nrow (:55).  get_data divides the reward by 5 (:71).
__device__ __forceinline__ float agent_step(int& x, int& y, int a, int gx, int gy, int nrow) {
    const int dist = abs(x - gx) + abs(y - gy);
    int dx, dy;
    move_of(a, dx, dy);
    x = min(max(x + dx, 0), nrow - 1);
    y = min(max(y + dy, 0), nrow - 1);
    const float rew = (dist == 0 && a == 0) ? 0.f : -(float)(dist + 1);
    return __fdiv_rn(rew, 5.f);
}

__global__ void __launch_bounds__(256) env_step_kernel(int32_t* __restrict__ state, const float* __restrict__ action,
                                                       const int32_t* __restrict__ desired, int n_envs, int n_agents,
                                                       int nrow, float* __restrict__ reward) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_envs * n_agents) return;
    const int ag = i % n_agents;
    int x = state[2 * i], y = state[2 * i + 1];
    reward[i] = agent_step(x, y, (int)action[i], desired[2 * ag], desired[2 * ag + 1], nrow);
    state[2 * i] = x;
    state[2 * i + 1] = y;
}

// Philox4x32-10 (Salmon et al.), counter-based: one call per (env, episode, step, agent)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}
__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }

// get_action (agents/resilient_CAC_agents.py:208-219) from three uniforms:
//   random_action = choice(n)            -> floor(u0 * n)
//   a_pol         = choice(n, p=probs)   -> searchsorted(cumsum(p)/sum, u1, 'right')
//   action        = choice([a_pol, random_action], p=[1-mu, mu]) -> a_pol if u2 < 1-mu else random_action
__device__ __forceinline__ int sample_action(const float (&p)[NACT], float u0, float u1, float u2, float one_minus_mu) {
    const int rand_a = min((int)(u0 * (float)NACT), NACT - 1);
    float cdf[NACT];
    float s = 0.f;
#pragma unroll
    for (int o = 0; o < NACT; ++o) { s += p[o]; cdf[o] = s; }
    int pol = 0;
#pragma unroll
    for (int o = 0; o < NACT; ++o) pol += (__fdiv_rn(cdf[o], s) <= u1) ? 1 : 0;
    pol = min(pol, NACT - 1);
    return u2 < one_minus_mu ? pol : rand_a;
}

template <int NA>
__global__ void __launch_bounds__(128) rollout_kernel(const __grid_constant__ rcmarl_rollout_args A) {
    extern __shared__ __align__(16) float smem[];
    constexpr int DIN = 2 * NA;
    constexpr int PA = param_count(DIN, NACT), PC = param_count(DIN, 1);
    constexpr int PAr = round4(PA), PCr = round4(PC);
    float* sa_w = smem;                 // [NA][PAr]
    float* sc_w = smem + NA * PAr;      // [NA][PCr]
    for (int i = threadIdx.x; i < NA * PA; i += blockDim.x) sa_w[(i / PA) * PAr + i % PA] = __ldg(A.actor_w + i);
    for (int i = threadIdx.x; i < NA * PC; i += blockDim.x) sc_w[(i / PC) * PCr + i % PC] = __ldg(A.critic_w + i);
    __syncthreads();

    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)A.n_episodes * A.n_envs;
    if (gid >= total) return;
    const int ep = (int)(gid / A.n_envs);
    const int env = (int)(gid - (int64_t)ep * A.n_envs);
    const uint64_t genv = (uint64_t)(A.env_offset + env);
    const uint64_t gep = (uint64_t)(A.episode_offset + ep);
    const uint2 key = make_uint2((uint32_t)A.seed, (uint32_t)(A.seed >> 32));
    const float one_minus_mu = 1.0f - A.mu;
    // agents nact .. NA-1 are unused slots of the instantiation (a team smaller than NA): they do not act, and their
    // state / action / reward columns are written as zeros (rcmarl/nets.py: the padded problem is the nact-agent problem)
    const int nact = (A.n_active > 0 && A.n_active < NA) ? A.n_active : NA;

    int px[NA], py[NA], gx[NA], gy[NA];
#pragma unroll
    for (int i = 0; i < NA; ++i) {
        gx[i] = A.desired[2 * i];
        gy[i] = A.desired[2 * i + 1];
        if (i >= nact) {
            px[i] = 0;
            py[i] = 0;
        } else if (A.init_state) {                                 // env.reset(), grid_world.py:37-45
            const int32_t* s0 = A.init_state + (((int64_t)ep * A.n_envs + env) * nact + i) * 2;
            px[i] = s0[0];
            py[i] = s0[1];
        } else {
            const uint4 rnd = philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)(genv >> 32) ^ 0x80000000u,
                                                       (uint32_t)gep, (uint32_t)i), key);
            px[i] = (int)__umulhi(rnd.x, (uint32_t)A.nrow);
            py[i] = (int)__umulhi(rnd.y, (uint32_t)A.ncol);
        }
    }
    float x[DIN];
#pragma unroll
    for (int i = 0; i < NA; ++i) {
        x[2 * i] = i < nact ? A.state_tab_x[px[i]] : 0.f;
        x[2 * i + 1] = i < nact ? A.state_tab_y[py[i]] : 0.f;
    }

    float* est = A.est + ((int64_t)ep * A.n_envs + env) * NA;
    float* retp = A.ret + ((int64_t)ep * A.n_envs + env) * NA;
    float ret[NA];
#pragma unroll 1
    for (int i = 0; i < NA; ++i) {                                 // train_agents.py:60-62
        float h1[HID], h2[HID];
        if (i >= nact) { est[i] = 0.f; continue; }
        features<DIN>(sc_w + i * PCr, x, h1, h2);
        est[i] = head1<DIN>(sc_w + i * PCr, h2);
    }
#pragma unroll
    for (int i = 0; i < NA; ++i) ret[i] = 0.f;

    float disc = 1.f;
    for (int j = 0; j < A.max_ep_len; ++j) {                       // train_agents.py:66-80
        const int64_t row = (A.time_begin + (int64_t)ep * A.max_ep_len + j) * A.n_envs + env;
        float* sa = A.sa + row * (3 * NA);
        float* ns = A.ns + row * (2 * NA);
        float* rr = A.r + row * NA;
        int act[NA];
#pragma unroll 1
        for (int i = 0; i < NA; ++i) {
            float h1[HID], h2[HID], p[NACT], mx, lse;
            if (i >= nact) { act[i] = 0; continue; }
            features<DIN>(sa_w + i * PAr, x, h1, h2);
            head5<DIN>(sa_w + i * PAr, h2, p);
            softmax5(p, mx, lse);
            float u0, u1, u2;
            if (A.uniforms) {
                const float* u = A.uniforms + ((((int64_t)ep * A.max_ep_len + j) * A.n_envs + env) * nact + i) * 3;
                u0 = u[0]; u1 = u[1]; u2 = u[2];
            } else {
                const uint4 rnd = philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)(genv >> 32), (uint32_t)gep,
                                                           (uint32_t)(j * NA + i)), key);
                u0 = u01(rnd.x); u1 = u01(rnd.y); u2 = u01(rnd.z);
            }
            act[i] = sample_action(p, u0, u1, u2, one_minus_mu);
        }
#pragma unroll
        for (int i = 0; i < NA; ++i) {                             // row: state and action (train_agents.py:76-79)
            sa[3 * i] = x[2 * i];
            sa[3 * i + 1] = x[2 * i + 1];
            sa[3 * i + 2] = (float)act[i];
        }
#pragma unroll
        for (int i = 0; i < NA; ++i) {                             // env.step + get_data
            float rew = agent_step(px[i], py[i], act[i], gx[i], gy[i], A.nrow);
            x[2 * i] = i < nact ? A.state_tab_x[px[i]] : 0.f;
            x[2 * i + 1] = i < nact ? A.state_tab_y[py[i]] : 0.f;
            rew = i < nact ? rew : 0.f;
            ns[2 * i] = x[2 * i];
            ns[2 * i + 1] = x[2 * i + 1];
            rr[i] = rew;
            ret[i] = fmaf(rew, disc, ret[i]);                      // train_agents.py:71
        }
        disc *= A.gamma;
    }
#pragma unroll
    for (int i = 0; i < NA; ++i) retp[i] = ret[i];
}

// Per-episode means over the environments of the logged quantities (train_agents.py:168-180 prints per-episode values; with
// N environments they become means, SURVEY Appendix C): out[ep][agent] = mean_e x[ep][e][agent], fixed-order tree.
__global__ void __launch_bounds__(256) episode_mean_kernel(const float* __restrict__ x, int n_envs, int n_agents,
                                                           float* __restrict__ out) {
    __shared__ float sh[256];
    const int ep = blockIdx.x, ag = blockIdx.y;
    const float* p = x + (int64_t)ep * n_envs * n_agents + ag;
    float s = 0.f;
    for (int e = threadIdx.x; e < n_envs; e += 256) s += p[(int64_t)e * n_agents];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[ep * n_agents + ag] = sh[0] / (float)n_envs;
}

template <int NA>
static int launch_rollout(const rcmarl_rollout_args& A, cudaStream_t st) {
    constexpr int DIN = 2 * NA;
    const size_t smem = sizeof(float) * NA * (round4(param_count(DIN, NACT)) + round4(param_count(DIN, 1)));
    if (smem > 48 * 1024)
        RC_CUDA(cudaFuncSetAttribute(rollout_kernel<NA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t total = (int64_t)A.n_episodes * A.n_envs;
    rollout_kernel<NA><<<(unsigned)((total + 127) / 128), 128, smem, st>>>(A);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

}  // namespace rcmarl

using namespace rcmarl;

extern "C" {

const char* rcmarl_version(void) { return "rcmarl-h100 0.1 (sm_90a, fp32)"; }

const char* rcmarl_status_string(int s) {
    switch (s) {
        case RCMARL_OK: return "ok";
        case RCMARL_ERR_ARG: return "invalid argument";
        case RCMARL_ERR_WORKSPACE: return "workspace too small";
        case RCMARL_ERR_CUDA: return "CUDA error";
        case RCMARL_ERR_NO_DEVICE: return "no CUDA device";
        default: return "unknown status";
    }
}

int rcmarl_last_cuda_error(void) { return last_cuda_error_get(); }

int rcmarl_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0, n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return RCMARL_ERR_NO_DEVICE;
    RC_CUDA(cudaGetDevice(&dev));
    if (sm_count) RC_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
    if (cc_major) RC_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    if (cc_minor) RC_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
    return RCMARL_OK;
}

int64_t rcmarl_param_count(int d_in, int n_out) { return param_count(d_in, n_out); }

int rcmarl_clip_mean(const float* vals, int n, int64_t P, int64_t row_stride, int H, float* out, void* stream) {
    if (!vals || !out || n < 1 || P < 0 || row_stride < P || H < 0 || H > RCMARL_MAX_H || H >= n) return RCMARL_ERR_ARG;
    if (P == 0) return RCMARL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    switch (H) {
        case 0: return launch_clip_mean<0>(vals, n, P, row_stride, out, st);
        case 1: return launch_clip_mean<1>(vals, n, P, row_stride, out, st);
        case 2: return launch_clip_mean<2>(vals, n, P, row_stride, out, st);
        case 3: return launch_clip_mean<3>(vals, n, P, row_stride, out, st);
        case 4: return launch_clip_mean<4>(vals, n, P, row_stride, out, st);
        case 5: return launch_clip_mean<5>(vals, n, P, row_stride, out, st);
        case 6: return launch_clip_mean<6>(vals, n, P, row_stride, out, st);
        default: return launch_clip_mean<7>(vals, n, P, row_stride, out, st);
    }
}

int rcmarl_rollout(const rcmarl_rollout_args* a, void* stream) {
    if (!a || !a->actor_w || !a->critic_w || !a->desired || !a->sa || !a->ns || !a->r || !a->est || !a->ret)
        return RCMARL_ERR_ARG;
    if (a->n_envs < 1 || a->n_episodes < 1 || a->max_ep_len < 1 || a->nrow < 1 || a->nrow > RCMARL_MAX_GRID ||
        a->ncol < 1 || a->ncol > RCMARL_MAX_GRID || a->time_begin < 0)
        return RCMARL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (a->n_agents == 5) return launch_rollout<5>(*a, st);
    if (a->n_agents == 16) return launch_rollout<16>(*a, st);
    return RCMARL_ERR_ARG;
}

int rcmarl_episode_means(const float* x, int n_episodes, int n_envs, int n_agents, float* out, void* stream) {
    if (!x || !out || n_episodes < 1 || n_envs < 1 || n_agents < 1 || n_agents > 65535) return RCMARL_ERR_ARG;
    episode_mean_kernel<<<dim3((unsigned)n_episodes, (unsigned)n_agents), 256, 0, (cudaStream_t)stream>>>(x, n_envs, n_agents, out);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_env_step(int32_t* state, const float* action, const int32_t* desired, int n_envs, int n_agents, int nrow,
                    float* reward_scaled, void* stream) {
    if (!state || !action || !desired || !reward_scaled || n_envs < 1 || n_agents < 1 || nrow < 1) return RCMARL_ERR_ARG;
    const int n = n_envs * n_agents;
    env_step_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(state, action, desired, n_envs, n_agents, nrow,
                                                                      reward_scaled);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

}  // extern "C"
