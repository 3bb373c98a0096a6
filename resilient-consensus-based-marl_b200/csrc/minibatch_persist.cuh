// minibatch_persist.cuh -- the adversaries' mini-batch fits as ONE persistent kernel per rcmarl_minibatch_sgd call
// (replaces critic.fit / TR.fit(batch_size=32, epochs=10) of agents/adversarial_CAC_agents.py:133,150,163,239,251).
//
// Round 1 ran every SGD step as two launches (grad_kernel + fused reduce / apply): 9 400 sequential steps per update
// round at ~17 us of launch gaps, prologues and a separate reduce grid each.  Here the CTAs stay resident for all
// epochs x mini-batches of a call, each chain's parameters live in the shared memory of its CTAs, and a step is
//   1. sweep this CTA's 64-row chunks of the mini-batch (GradCore, register accumulators),
//   2. fixed-order CTA reduction; the CTA's sums go out as level-1 cells {value, seq} (8-byte stores),
//   3. the CTAs of a chain split the parameters into slices: the owner of a slice polls the level-1 cells of all CTAs
//      of its chain for that slice, adds them in CTA order and publishes level-2 cells -- into its own GPU's buffer, or
//      (data parallel) into EVERY rank's buffer over NVLink peer memory (comm.cuh, same cell format),
//   4. every CTA polls the level-2 cells of all parameters (rank-ordered sum over the ranks) and applies the SGD step to
//      its shared-memory copy of the chain's parameters.
// No grid barrier, no atomics, no launches, no host round trip; every sum has a fixed association, so the result is
// bitwise reproducible and identical on every CTA and every rank.  A sequence number is used exactly once per step, so
// stale cells can never be mistaken for fresh ones; the cell buffers must start zeroed (sequence numbers start at 1).
// Why single-buffered level-1 cells are safe: a CTA writes its level-1 cells of step s+1 only after it has read all
// level-2 cells of step s, which exist only after every slice owner of its chain has read the level-1 cells of step s.
// Level-2 cells are double-buffered by sequence parity for the cross-rank case (comm.cuh).
#pragma once
#include "grad_kernel.cuh"
#include "comm.cuh"

namespace rcmarl {

struct MbChain {
    float* w;                    // packed parameters, updated in place (read at start, written back at the end)
    const float* target;
    const int32_t* time_idx;     // [epochs][n_times] shuffled time rows
    float* loss_out;             // += loss_coef * sum over the first epoch's steps of sum e^2 (may be null)
    int64_t target_stride;
    float lr, loss_coef;
    int32_t kind, loss_accumulate;
};

struct MbParams {
    rcmarl_rows rows;                       // sa / ns / r, row_begin, n_envs, n_agents (n_rows, time_idx set per step)
    MbChain chains[RCMARL_MAX_JOBS];
    int16_t cta_first[RCMARL_MAX_JOBS + 1];
    int32_t n_chains, epochs, n_times, mb_times, stride;
    uint2* cells1;                          // level 1: [n_ctas][stride]
    uint32_t seq1;                          // level-1 sequence number of the call's first step
    CommDev comm;                           // level 2 (world == 1: cells[0] is a local buffer); comm.seq = first step's
};

__device__ __forceinline__ uint2 poll_cell(const uint2* cell, uint32_t seq, uint32_t* err) {
    uint2 x = ld_cell(cell);
    if (x.y != seq) {
        const long long t0 = clock64();
        do {
            if (clock64() - t0 > 40000000000LL) {      // ~20 s: fail loudly instead of hanging the GPU
                if (err) *err = 2u;
                __threadfence_system();
                __trap();
            }
            __nanosleep(RCMARL_CELL_POLL_NS);           // spinning CTAs must not crowd the writers out of the L2 queues
            x = ld_cell(cell);
        } while (x.y != seq);
    }
    return x;
}

template <int NA, int DIN, int NW>
__device__ __forceinline__ void mb_body(const MbParams& P, const MbChain& ch, int j, float* smem, int y, int gy) {
    using Core = GradCore<NA, DIN, 1, NW>;
    constexpr int NP = Core::NP;
    Core core;
    core.setup(smem);
    pdl_wait();
    stage_weights(core.sw, ch.w, NP);
    __syncthreads();
    core.write_pads();

    rcmarl_grad_job gj;
    gj.w = ch.w; gj.target = ch.target; gj.sums = nullptr; gj.time_idx = nullptr;
    gj.target_stride = ch.target_stride; gj.kind = ch.kind; gj.action_agent = 0;
    rcmarl_rows Rw = P.rows;

    const int cta = blockIdx.x;
    uint2* my1 = P.cells1 + (int64_t)cta * P.stride;
    const uint2* chain1 = P.cells1 + (int64_t)P.cta_first[j] * P.stride;
    // slice of this CTA: entries [sl_begin, sl_end) of the NP + 1 sums (the last entry is the loss)
    const int per = (NP + 1 + gy - 1) / gy;
    const int sl_begin = y * per < NP + 1 ? y * per : NP + 1;
    const int sl_end = sl_begin + per < NP + 1 ? sl_begin + per : NP + 1;
    // level-1 gather geometry: S lanes share an entry (S = power of two >= min(gy, 32)), each adds every S-th CTA
    int S = 1;
    while (S < gy && S < 32) S <<= 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sgroup = lane & (S - 1), e_local = lane / S, e_per_warp = 32 / S;
    const int64_t off2 = (int64_t)j * P.stride;
    const CommDev& comm = P.comm;
    uint32_t seq2 = P.comm.seq;
    const int nb = (P.n_times + P.mb_times - 1) / P.mb_times;
    uint32_t seq1 = P.seq1;
    float loss_acc = 0.f;

    for (int e = 0; e < P.epochs; ++e) {
        for (int b = 0; b < nb; ++b, ++seq1, ++seq2) {
            const int cnt = P.n_times - b * P.mb_times < P.mb_times ? P.n_times - b * P.mb_times : P.mb_times;
            Rw.n_rows = (int64_t)cnt * Rw.n_envs;
            Rw.time_idx = ch.time_idx + (int64_t)e * P.n_times + (int64_t)b * P.mb_times;
            core.zero_acc();
            core.sweep(Rw, gj, y, gy);
            // ---- level 1: this CTA's sums
            const uint32_t s1 = seq1;
            core.cta_reduce([my1, s1](int i, float v) { st_cell(my1 + i, v, s1); });
            // ---- slice owner: CTA-ordered sum over the chain's CTAs, publish level 2
            for (int base = sl_begin + warp * e_per_warp; base < sl_end; base += NW * e_per_warp) {
                const int i = base + e_local;
                float s = 0.f;
                if (i < sl_end) {
                    for (int yy = sgroup; yy < gy; yy += S)
                        s += __uint_as_float(poll_cell(chain1 + (int64_t)yy * P.stride + i, s1, comm.error).x);
                }
                for (int o = 1; o < S; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (i < sl_end && sgroup == 0) comm_push(comm, off2 + i, s, seq2);
            }
            // ---- level 2: every CTA applies the step to its own copy (tile region is free: cta_reduce is done with it)
            const float coef = ch.lr * 2.0f / ((float)Rw.n_rows * (float)comm.world);
            for (int i = threadIdx.x; i <= NP; i += blockDim.x) {
                const float tot = comm_wait_total(comm, off2 + i, seq2);
                if (i < NP) core.sw[i] = core.sw[i] - coef * tot;
                else if (e == 0) loss_acc += ch.loss_coef * tot;
            }
            __syncthreads();                 // new parameters visible to all warps; tile region reusable
            core.write_pads();
        }
    }
    if (y == 0) {
        for (int i = threadIdx.x; i < NP; i += blockDim.x) ch.w[i] = core.sw[i];
        if (threadIdx.x == (NP % blockDim.x) && ch.loss_out) *ch.loss_out = ch.loss_accumulate ? *ch.loss_out + loss_acc : loss_acc;
    }
}

template <int NA>
__global__ void __launch_bounds__(32 * grad_warps<NA, RCMARL_LOSS_MSE>(), 1)
mb_persist_kernel(const __grid_constant__ MbParams P) {
    extern __shared__ __align__(16) float smem[];
    constexpr int NW = grad_warps<NA, RCMARL_LOSS_MSE>();
    pdl_launch_dependents();         // the next kernel may be queued; it waits for this grid with griddepcontrol.wait
    int j = 0;
    while (j + 1 < P.n_chains && (int)blockIdx.x >= P.cta_first[j + 1]) ++j;
    const MbChain& ch = P.chains[j];
    const int y = (int)blockIdx.x - P.cta_first[j], gy = P.cta_first[j + 1] - P.cta_first[j];
    if (ch.kind == RCMARL_IN_SA) mb_body<NA, 3 * NA, NW>(P, ch, j, smem, y, gy);
    else mb_body<NA, 2 * NA, NW>(P, ch, j, smem, y, gy);
}

}  // namespace rcmarl
