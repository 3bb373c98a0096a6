// grad_kernel.cuh -- fused forward + backward of the 20-wide RPBCAC MLPs over a set of buffer rows
// (rcmarl_grad, include/rcmarl.h; replaces the fwd/bwd inside critic.fit / TR.fit / actor.train_on_batch,
// agents/resilient_CAC_agents.py:99,118,136 and adversarial:41,116,133,150,163).
//
// The kernel is FP32-FMA work fed from shared memory, and the shared-memory pipe (one wavefront per clock per SM) is
// the first limit: a warp-uniform LDS.128 costs 2 wavefronts and any other LDS.128 costs 4, while the four FMA pipes
// retire 4 warp-FFMAs per clock.  Balance
// therefore needs >= 4 FFMA per wavefront everywhere:
//   phase 1 (forward + backward-data): every lane carries R = 2 buffer rows, so each broadcast weight quad
//            (uniform LDS.128, 2 wavefronts) feeds 8 FFMA;
//   phase 2 (weight gradients = sum over rows of outer products): the per-row activation / delta vectors are
//            staged in a warp-private shared-memory tile and every lane owns one 8x8 register tile of the
//            gradient (4 LDS.128 = 16 wavefronts per 64 FFMA); lanes are split into row groups so that
//            NG x (number of tiles) <= 32 lanes are busy.  Accumulators stay in registers across ALL rows of the
//            CTA; the output-layer gradient of the scalar nets is accumulated per lane in phase 1.
// Reductions are fixed-order (lane -> warp -> CTA partial -> reduce_kernel): bitwise reproducible.
#pragma once
#include "common.cuh"

namespace rcmarl {

__host__ __device__ constexpr int round8(int n) { return (n + 7) & ~7; }

template <int DIN, int NOUT>
struct TileLayout {
    static constexpr bool L3T = (NOUT > 1);             // output-layer gradient through tiles (actor) or per lane
    static constexpr int LA1 = round8(DIN + 1);         // [x .. , 1, 0 pad]
    static constexpr int OA1 = 0;
    static constexpr int OA2 = LA1;                     // [h1(20), 1, 0, 0, 0]
    static constexpr int OA3 = OA2 + 24;                // [h2(20), 1, 0, 0, 0]   (only if L3T)
    static constexpr int OD1 = OA3 + (L3T ? 24 : 0);    // delta1 (20) + 4 zeros
    static constexpr int OD2 = OD1 + 24;                // delta2 (20) + 4 zeros
    static constexpr int OD3 = OD2 + 24;                // dLoss/dlogits (NOUT) + zeros (only if L3T)
    static constexpr int RAW = OD3 + (L3T ? 8 : 0);
    // row stride: odd number of 16-byte units => conflict-free float4 stores within a quarter-warp
    static constexpr int RS = ((RAW / 4) % 2 == 0) ? RAW + 4 : RAW;
    static constexpr int NT1 = (LA1 / 8) * 3;
    static constexpr int NT2 = 9;
    static constexpr int NT3 = L3T ? 3 : 0;
    static constexpr int NT = NT1 + NT2 + NT3;          // 8x8 tiles covering all weight gradients
    static_assert(NT <= 32, "tile count exceeds a warp");
    static constexpr int NG = 32 / NT;                  // row groups processed concurrently by one warp
    static constexpr int ROWS = 64;                     // rows per warp chunk (R = 2 per lane)

    __device__ static __forceinline__ void tile_offsets(int t, int& aoff, int& doff) {
        if (t < NT1) {
            aoff = OA1 + 8 * (t / 3); doff = OD1 + 8 * (t % 3);
        } else if (t < NT1 + NT2) {
            t -= NT1; aoff = OA2 + 8 * (t / 3); doff = OD2 + 8 * (t % 3);
        } else {
            t -= NT1 + NT2; aoff = OA3 + 8 * t; doff = OD3;
        }
    }
    // packed-parameter index of element (ii, jj) of tile t, -1 for padding
    __device__ static __forceinline__ int tile_param(int t, int ii, int jj) {
        if (t < NT1) {
            const int i = 8 * (t / 3) + ii, j = 8 * (t % 3) + jj;
            if (j >= HID) return -1;
            return i < DIN ? i * HID + j : (i == DIN ? off_b1(DIN) + j : -1);
        } else if (t < NT1 + NT2) {
            t -= NT1;
            const int i = 8 * (t / 3) + ii, j = 8 * (t % 3) + jj;
            if (j >= HID) return -1;
            return i < HID ? off_W2(DIN) + i * HID + j : (i == HID ? off_b2(DIN) + j : -1);
        } else if (t < NT) {
            t -= NT1 + NT2;
            const int i = 8 * t + ii, o = jj;
            if (o >= NOUT) return -1;
            return i < HID ? off_W3(DIN) + i * NOUT + o : (i == HID ? off_b3(DIN, NOUT) + o : -1);
        }
        return -1;
    }
};

constexpr int GRAD_SMEM_BUDGET = 227 * 1024;   // one CTA per SM (up to 255 registers per thread)
// staged input rows: 64 buffer rows of sa (3*NA floats) or ns (2*NA floats); the staging buffer is sized for sa rows:
// 3*NA == DIN for the team-reward net (DIN = 3*NA) and 3*DIN/2 for critic / actor (DIN = 2*NA)
__host__ __device__ constexpr int stage_floats_per_row(int din, bool is_sa_net) { return is_sa_net ? din : (3 * din) / 2; }

// warps per CTA: as many 64-row tiles as fit next to the staged weights, at most 8
// Bulk-copy input staging costs 64 x 3*NA x 4 bytes of shared memory per warp.  At n_agents = 5 (3.8 KB per warp) it fits
// next to 8 tiles; at n_agents = 16 it would cut the CTA from 6 to 4 warps, so those instantiations keep per-lane loads.
__host__ __device__ constexpr bool grad_use_tma(int na) { return na <= 5; }

template <int DIN, int NOUT, bool SA_NET>
constexpr int grad_warps_for() {
    using L = TileLayout<DIN, NOUT>;
    const int na = SA_NET ? DIN / 3 : DIN / 2;
    const int avail = GRAD_SMEM_BUDGET - 4 * (round4(param_count(DIN, NOUT)) + 16) - 128;
    const int n = avail / (4 * L::ROWS * L::RS + (grad_use_tma(na) ? 4 * L::ROWS * stage_floats_per_row(DIN, SA_NET) : 0));
    return n > 8 ? 8 : n;
}
template <int NA, int LOSS>
constexpr int grad_warps() {
    if (LOSS == RCMARL_LOSS_CE) return grad_warps_for<2 * NA, NACT, false>();
    const int a = grad_warps_for<3 * NA, 1, true>(), b = grad_warps_for<2 * NA, 1, false>();
    return a < b ? a : b;
}

// Relative cost of one buffer row for a job (FMA issue slots per lane-row): phase 1 (forward, output layer, backward-data)
// plus phase 2 (the NT 8x8 tiles are spread over NG row groups, so a 64-row chunk takes 64 / NG tile steps of 64 FMA).
__host__ __device__ constexpr int grad_row_cost(int din, int nout) {
    const int la1 = round8(din + 1);
    const int nt = (la1 / 8) * 3 + 9 + (nout > 1 ? 3 : 0);
    const int ng = 32 / nt;
    return din * HID + 2 * HID * HID + 2 * HID * nout + 2048 / ng;
}

// ---- 1-D bulk copy (TMA engine, SASS UBLKCP) of the next chunk's input rows into a warp-private staging buffer ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}

struct GradParams {
    rcmarl_rows rows;
    rcmarl_grad_job jobs[RCMARL_MAX_JOBS];
    float* partial;   // [CTA][stride]: one slot per CTA of the 1-D grid
    int32_t n_jobs;
    int32_t stride;
    // job j owns the CTAs [cta_first[j], cta_first[j + 1]) of the 1-D grid (train_kernels.cu, plan_grid)
    int16_t cta_first[RCMARL_MAX_JOBS + 1];
};

__device__ __forceinline__ void st4(float* p, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}

// GradCore: the per-CTA machinery of the fused forward + backward pass, split into set-up (once per kernel), the row
// sweep (register accumulators) and the fixed-order CTA reduction, so that the one-shot kernel (grad_kernel) and the
// persistent mini-batch kernel (minibatch_persist.cuh) share one body.  All members live in registers (everything is
// force-inlined and fully unrolled).
template <int NA, int DIN, int NOUT, int GRAD_WARPS>
struct GradCore {
    using L = TileLayout<DIN, NOUT>;
    static constexpr int NP = param_count(DIN, NOUT);
    static constexpr int R = 2;
    static constexpr int SROW = 3 * NA;                                     // staged row = one sa row (ns rows are shorter)
    static constexpr int SWARP = grad_use_tma(NA) ? L::ROWS * SROW : 0;      // staging floats per warp

    float* sw;          // staged network parameters (shared)
    float* tiles;       // [GRAD_WARPS][ROWS][RS]
    float* wt;          // this warp's tile
    float* stage;       // this warp's bulk-copy staging buffer
    uint64_t* bar;      // this warp's mbarrier
    int warp, lane;
    uint32_t phase;
    // phase-2 assignment of this lane: tile `tile`, row group `grp`
    int grp, aoff, doff;
    f2 acc[32];                            // 8x8 tile, packed as pairs over the delta index
    float g3[L::L3T ? 1 : HID + 1];       // scalar nets: output-layer gradient per lane [W3(20) | b3]
    float loss;

    // shared-memory carve-up + mbarrier init; nothing here touches global memory (may run before pdl_wait)
    __device__ __forceinline__ void setup(float* smem) {
        sw = smem;
        tiles = smem + round4(NP);
        warp = threadIdx.x >> 5;
        lane = threadIdx.x & 31;
        wt = tiles + warp * (L::ROWS * L::RS);
        stage = tiles + GRAD_WARPS * (L::ROWS * L::RS) + warp * SWARP;
        bar = reinterpret_cast<uint64_t*>(tiles + GRAD_WARPS * (L::ROWS * L::RS) + GRAD_WARPS * SWARP) + warp;
        phase = 0;
        if (lane == 0) {
            mbar_init(bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        const bool busy = lane < L::NG * L::NT;
        const int tile = busy ? lane % L::NT : 0;
        grp = busy ? lane / L::NT : 0;
        L::tile_offsets(tile, aoff, doff);
    }

    // the constant columns of this lane's two tile rows ([.., 1, 0 pad] of the activations, zero pad of the deltas)
    // never change: write them once instead of once per chunk (saves 3-4 of 22 STS.128 per row).  Must be repeated after
    // cta_reduce (which reuses the tiles).
    __device__ __forceinline__ void write_pads() {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            float* rowp = wt + (lane + 32 * r) * L::RS;
#pragma unroll
            for (int q = 0; q < L::LA1 / 4; ++q)
                if (4 * q >= DIN) st4(rowp + L::OA1 + 4 * q, 4 * q == DIN ? 1.f : 0.f, 0.f, 0.f, 0.f);
            st4(rowp + L::OA2 + 20, 1.f, 0.f, 0.f, 0.f);
            if constexpr (L::L3T) st4(rowp + L::OA3 + 20, 1.f, 0.f, 0.f, 0.f);
            st4(rowp + L::OD1 + 20, 0.f, 0.f, 0.f, 0.f);
            st4(rowp + L::OD2 + 20, 0.f, 0.f, 0.f, 0.f);
        }
        __syncwarp();
    }

    __device__ __forceinline__ void zero_acc() {
#pragma unroll
        for (int e = 0; e < 32; ++e) acc[e] = pack2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < (L::L3T ? 1 : HID + 1); ++j) g3[j] = 0.f;
        loss = 0.f;
    }

    // Sweep the rows of `Rw` that belong to CTA y of gy (64-row chunks, see below); weights are read from `sw`.
    // Accumulates into acc / g3 / loss.
    __device__ __forceinline__ void sweep(const rcmarl_rows& Rw, const rcmarl_grad_job& job, int y, int gy) {
    // Input staging by the TMA engine: the 64 rows of a chunk are one contiguous, 16-byte aligned span of sa / ns whenever
    // the chunk is full and (contiguous row mode, or gathered mode with n_envs % 64 == 0); lane 0 issues one 1-D bulk copy
    // per chunk, completion is tracked by the warp's mbarrier; other chunks fall back to per-lane loads.
    const bool from_ns = (DIN == 2 * NA) && job.kind == RCMARL_IN_NS;
    const int rowf = from_ns ? 2 * NA : 3 * NA;
    const float* in_base = from_ns ? Rw.ns : Rw.sa;
    const bool gather_ok = grad_use_tma(NA) && ((Rw.time_idx == nullptr) || (Rw.n_envs % L::ROWS == 0));
    auto stage_src = [&](int64_t c, const float*& src) -> bool {
        if (!gather_ok || (c + 1) * L::ROWS > Rw.n_rows) return false;
        src = in_base + row_of(Rw, c * L::ROWS) * rowf;
        return (reinterpret_cast<uintptr_t>(src) & 15) == 0;
    };
    bool staged = false;
    // Chunk c of the job goes to (CTA y, warp w) with c = k * cstep + w * gy + y: warp-major, so that the last, partial
    // round leaves one or two busy warps on every SM (on different schedulers, so they run faster alone).  A CTA-major
    // order (c = k * cstep + y * GRAD_WARPS + w) would leave a few SMs with all warps busy and the others idle, and the
    // whole launch would wait for a full extra round on those SMs.
    const int64_t cstep = (int64_t)gy * GRAD_WARPS;
    const int64_t cfirst = (int64_t)warp * gy + y;
    {
        const int64_t c0 = cfirst;
        const float* src = nullptr;
        if (c0 * L::ROWS < Rw.n_rows) staged = stage_src(c0, src);
        if (staged && lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic accesses of the buffer
            bulk_load(stage, src, (uint32_t)(L::ROWS * rowf * sizeof(float)), bar);
        }
    }
    const int64_t nchunks = (Rw.n_rows + L::ROWS - 1) / L::ROWS;
    for (int64_t c = cfirst; c < nchunks; c += cstep) {
        // ---------------- phase 1: two rows per lane (lane, lane + 32 of the chunk) ----------------
        {
            bool live[R];
            int64_t row[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int64_t m = c * L::ROWS + lane + 32 * r;
                live[r] = m < Rw.n_rows;
                row[r] = row_of(Rw, live[r] ? m : 0);      // dead rows read row 0 and contribute zeros
            }
            float h1[R][HID], h2[R][HID];
            {
                float x[R][DIN];
                if (staged) {                                              // rows of this chunk were bulk-copied
                    mbar_wait(bar, phase);
                    phase ^= 1u;
                    const int skip = (DIN == 2 * NA && !from_ns) ? 1 : 0;  // s out of sa: skip the action slots
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        const float* sp = stage + (lane + 32 * r) * rowf;
#pragma unroll
                        for (int k = 0; k < DIN; ++k) x[r][k] = sp[k + skip * (k >> 1)];
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < R; ++r) load_x<NA, DIN>(Rw, job.kind, row[r], x[r]);
                }
                __syncwarp();
                {                                                          // prefetch the next chunk of this warp
                    const int64_t c2 = c + cstep;
                    const float* src = nullptr;
                    staged = (c2 < nchunks) && stage_src(c2, src);
                    if (staged && lane == 0) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads before async writes
                        bulk_load(stage, src, (uint32_t)(L::ROWS * rowf * sizeof(float)), bar);
                    }
                }
                dense20_rows<DIN, R>(sw, sw + off_b1(DIN), x, h1);
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    float* a1 = wt + (lane + 32 * r) * L::RS + L::OA1;
#pragma unroll
                    for (int q = 0; q < L::LA1 / 4; ++q) {
                        if (4 * q >= DIN) continue;                       // constant columns: write_pads()
                        float v[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int k = 4 * q + u;
                            v[u] = k < DIN ? x[r][k < DIN ? k : 0] : (k == DIN ? 1.f : 0.f);
                        }
                        st4(a1 + 4 * q, v[0], v[1], v[2], v[3]);
                    }
                }
            }
            dense20_rows<HID, R>(sw + off_W2(DIN), sw + off_b2(DIN), h1, h2);
            float d2[R][HID];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                float* rowp = wt + (lane + 32 * r) * L::RS;
#pragma unroll
                for (int q = 0; q < 5; ++q) st4(rowp + L::OA2 + 4 * q, h1[r][4 * q], h1[r][4 * q + 1], h1[r][4 * q + 2], h1[r][4 * q + 3]);
                const float tgt = live[r] ? __ldg(job.target + row[r] * job.target_stride) : 0.f;
                if constexpr (NOUT == 1) {
                    // Keras MSE (Appendix A.2): dLoss/dout = 2 (out - y) / B; the 2/B is applied by the caller
                    const float e = live[r] ? head1<DIN>(sw, h2[r]) - tgt : 0.f;
                    loss = fmaf(e, e, loss);
#pragma unroll
                    for (int j = 0; j < HID; ++j) {
                        g3[j] = fmaf(h2[r][j], e, g3[j]);
                        d2[r][j] = sw[off_W3(DIN) + j] * e * lrelu_grad_from_out(h2[r][j]);
                    }
                    g3[HID] += e;
                } else {
                    // weighted sparse categorical cross-entropy on the logits (Appendix A.5)
                    float p[NACT], mx, lse, g[NACT];
                    head5<DIN>(sw, h2[r], p);
                    const int a = (int)__ldg(Rw.sa + row[r] * (3 * NA) + 3 * job.action_agent + 2);
                    float la = 0.f;
#pragma unroll
                    for (int o = 0; o < NACT; ++o) la = (o == a) ? p[o] : la;
                    softmax5(p, mx, lse);
                    loss = fmaf(tgt, (mx + lse) - la, loss);
#pragma unroll
                    for (int o = 0; o < NACT; ++o) g[o] = (p[o] - (o == a ? 1.f : 0.f)) * tgt;
#pragma unroll
                    for (int q = 0; q < 5; ++q) st4(rowp + L::OA3 + 4 * q, h2[r][4 * q], h2[r][4 * q + 1], h2[r][4 * q + 2], h2[r][4 * q + 3]);
                    st4(rowp + L::OD3, g[0], g[1], g[2], g[3]);
                    st4(rowp + L::OD3 + 4, g[4], 0.f, 0.f, 0.f);
#pragma unroll
                    for (int j = 0; j < HID; ++j) {
                        float s = 0.f;
#pragma unroll
                        for (int o = 0; o < NACT; ++o) s = fmaf(sw[off_W3(DIN) + j * NACT + o], g[o], s);
                        d2[r][j] = s * lrelu_grad_from_out(h2[r][j]);
                    }
                }
#pragma unroll
                for (int q = 0; q < 5; ++q) st4(rowp + L::OD2 + 4 * q, d2[r][4 * q], d2[r][4 * q + 1], d2[r][4 * q + 2], d2[r][4 * q + 3]);
            }
            // delta1[i] = (W2[i][:] . delta2) * lrelu'(z1[i]) for both rows; each W2 quad feeds 8 FFMA
            f2 d2p[R][HID / 2];
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int j = 0; j < HID / 2; ++j) d2p[r][j] = pack2(d2[r][2 * j], d2[r][2 * j + 1]);
#pragma unroll
            for (int q = 0; q < 5; ++q) {
                float d1[R][4];
#pragma unroll
                for (int ii = 0; ii < 4; ++ii) {
                    const int i = 4 * q + ii;
                    f2 s[R];
#pragma unroll
                    for (int r = 0; r < R; ++r) s[r] = pack2(0.f, 0.f);
#pragma unroll
                    for (int qq = 0; qq < 5; ++qq) {
                        const float4 v = *reinterpret_cast<const float4*>(sw + off_W2(DIN) + i * HID + 4 * qq);
                        const f2 w0 = pack2(v.x, v.y), w1 = pack2(v.z, v.w);
#pragma unroll
                        for (int r = 0; r < R; ++r) {
                            s[r] = fma2(w0, d2p[r][2 * qq], s[r]);
                            s[r] = fma2(w1, d2p[r][2 * qq + 1], s[r]);
                        }
                    }
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        float se, so;
                        unpack2(s[r], se, so);
                        d1[r][ii] = (se + so) * lrelu_grad_from_out(h1[r][i]);
                    }
                }
#pragma unroll
                for (int r = 0; r < R; ++r)
                    st4(wt + (lane + 32 * r) * L::RS + L::OD1 + 4 * q, d1[r][0], d1[r][1], d1[r][2], d1[r][3]);
            }
        }
        __syncwarp();
        // ---------------- phase 2: 8x8 register tile per lane, NG rows per step ----------------
        constexpr int kPh2Unroll = 4;
#pragma unroll kPh2Unroll
        for (int it = 0; it < L::ROWS / L::NG; ++it) {
            const float* rp = wt + (it * L::NG + grp) * L::RS;
            const float4 a0 = *reinterpret_cast<const float4*>(rp + aoff);
            const float4 a1 = *reinterpret_cast<const float4*>(rp + aoff + 4);
            const float4 d0 = *reinterpret_cast<const float4*>(rp + doff);
            const float4 d1 = *reinterpret_cast<const float4*>(rp + doff + 4);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const f2 d[4] = {pack2(d0.x, d0.y), pack2(d0.z, d0.w), pack2(d1.x, d1.y), pack2(d1.z, d1.w)};
#pragma unroll
            for (int ii = 0; ii < 8; ++ii) {
                const f2 aa = pack2(a[ii], a[ii]);
#pragma unroll
                for (int jp = 0; jp < 4; ++jp) acc[ii * 4 + jp] = fma2(aa, d[jp], acc[ii * 4 + jp]);
            }
        }
        __syncwarp();
    }

    }

    // CTA reduction in fixed order (bitwise reproducible): store(i, v) receives this CTA's gradient sums for the packed
    // parameters i = 0 .. NP-1 and the loss sum as i = NP (each index exactly once, from some thread).
    // Reuses the tile region (call write_pads() before the next sweep).  All threads must call it.
    template <class ST>
    __device__ __forceinline__ void cta_reduce(ST store) {
    __syncthreads();
    float* red = tiles;                               // [GRAD_WARPS][32][64]
    {
        float4* dst = reinterpret_cast<float4*>(red + (warp * 32 + lane) * 64);
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            float4 v;
            unpack2(acc[2 * q], v.x, v.y);
            unpack2(acc[2 * q + 1], v.z, v.w);
            dst[q] = v;
        }
    }
    float* red3 = red + GRAD_WARPS * 32 * 64;         // [GRAD_WARPS][HID + 2]: lane-private layer-3 sums + loss
    loss = warp_sum(loss);
    if (lane == 0) red3[warp * (HID + 2) + HID + 1] = loss;
    if constexpr (!L::L3T) {
#pragma unroll
        for (int j = 0; j <= HID; ++j) {
            const float s = warp_sum(g3[j]);
            if (lane == 0) red3[warp * (HID + 2) + j] = s;
        }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < L::NT * 64; q += blockDim.x) {
        const int t = q >> 6, e = q & 63;
        const int idx = L::tile_param(t, e >> 3, e & 7);
        if (idx >= 0) {
            float s = 0.f;
            for (int w = 0; w < GRAD_WARPS; ++w)
#pragma unroll
                for (int g = 0; g < L::NG; ++g) s += red[(w * 32 + g * L::NT + t) * 64 + e];
            store(idx, s);
        }
    }
    if constexpr (!L::L3T) {
        if (threadIdx.x <= HID) {
            float s = 0.f;
            for (int w = 0; w < GRAD_WARPS; ++w) s += red3[w * (HID + 2) + threadIdx.x];
            store((threadIdx.x < HID ? off_W3(DIN) : off_b3(DIN, 1) - HID) + threadIdx.x, s);
        }
    }
    if (threadIdx.x == 32) {
        float s = 0.f;
        for (int w = 0; w < GRAD_WARPS; ++w) s += red3[w * (HID + 2) + HID + 1];
        store(NP, s);
    }
    }
};

// y / gy: index of this CTA among the gy CTAs of its job
template <int NA, int DIN, int NOUT, int GRAD_WARPS>
__device__ __forceinline__ void grad_body(const GradParams& P, const rcmarl_grad_job& job, float* smem, int y, int gy) {
    GradCore<NA, DIN, NOUT, GRAD_WARPS> core;
    rcmarl_rows Rw = P.rows;
    if (job.time_idx) Rw.time_idx = job.time_idx;
    core.setup(smem);
    pdl_wait();                       // everything above overlaps the tail of the previous kernel (PDL)
    stage_weights(core.sw, job.w, core.NP);
    __syncthreads();
    core.write_pads();
    core.zero_acc();
    core.sweep(Rw, job, y, gy);
    // a reduce kernel launched as a programmatic dependent (reduce_partials, train_kernels.cu) is queued once every CTA is
    // past its row loop, i.e. before the last CTA exits; it waits for this grid with griddepcontrol.wait
    pdl_launch_dependents();
    float* out = P.partial + (int64_t)blockIdx.x * P.stride;
    core.cta_reduce([out](int i, float v) { out[i] = v; });
}

template <int NA, int LOSS>
__global__ void __launch_bounds__(32 * grad_warps<NA, LOSS>(), 1) grad_kernel(const __grid_constant__ GradParams P) {
    extern __shared__ __align__(16) float smem[];
    constexpr int NW = grad_warps<NA, LOSS>();
    int j = 0;
    while (j + 1 < P.n_jobs && (int)blockIdx.x >= P.cta_first[j + 1]) ++j;
    const rcmarl_grad_job& job = P.jobs[j];
    const int y = (int)blockIdx.x - P.cta_first[j], gy = P.cta_first[j + 1] - P.cta_first[j];
    if (LOSS == RCMARL_LOSS_CE) {
        grad_body<NA, 2 * NA, NACT, NW>(P, job, smem, y, gy);
    } else if (job.kind == RCMARL_IN_SA) {
        grad_body<NA, 3 * NA, 1, NW>(P, job, smem, y, gy);
    } else {
        grad_body<NA, 2 * NA, 1, NW>(P, job, smem, y, gy);
    }
}

template <int NA, int DIN, int NOUT, int NW>
constexpr int grad_smem_floats() {
    using L = TileLayout<DIN, NOUT>;
    constexpr int tiles = NW * L::ROWS * L::RS;
    constexpr int red = NW * 32 * 64 + NW * (HID + 2);
    static_assert(tiles >= red, "the CTA reduction buffer reuses the tile region");
    constexpr int stage = (grad_use_tma(NA) ? NW * L::ROWS * 3 * NA : 0) + 2 * NW + 8;   // staged rows + one mbarrier per warp
    return round4(param_count(DIN, NOUT)) + tiles + stage + 16;
}

// dynamic shared memory of grad_kernel<NA, LOSS> (and of mb_persist_kernel<NA>, LOSS = MSE): one launch serves every job
// kind of its loss, so MSE takes the larger of the SA-net and S-net layouts
template <int NA, int LOSS>
constexpr size_t grad_smem_bytes() {
    constexpr int NW = grad_warps<NA, LOSS>();
    if constexpr (LOSS == RCMARL_LOSS_CE) {
        return sizeof(float) * grad_smem_floats<NA, 2 * NA, NACT, NW>();
    } else {
        constexpr int sa = grad_smem_floats<NA, 3 * NA, 1, NW>(), s = grad_smem_floats<NA, 2 * NA, 1, NW>();
        return sizeof(float) * (sa > s ? sa : s);
    }
}

}  // namespace rcmarl
