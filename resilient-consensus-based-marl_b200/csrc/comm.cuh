// comm.cuh -- one-shot all-reduce over NVLink peer memory, fused into the reduction / apply kernels
// (data-parallel env shards, SURVEY 8e).  Every rank owns one cudaMalloc'ed exchange buffer that all peers map
// through CUDA IPC:  [ cells: 2 slots x world sources x max_floats x {value, seq} | error word ].
//
// Low-latency ("LL") push protocol for step `seq` (identical call sequence on every rank):
//   1. the thread that owns element e of the rank's local sums STORES the 8-byte cell {value bits, seq} into slot
//      (seq & 1), source `rank`, element e of EVERY peer's buffer (own included) with one aligned 8-byte store per peer:
//      value and sequence number travel in the same NVLink write, so no fence, no separate flag and no second
//      round trip is needed (the 8-byte store is single-copy atomic);
//   2. the same thread polls the `world` cells of element e in its OWN buffer (local memory, ld.volatile) until each
//      shows `seq`, and adds the values in rank order, so all ranks obtain bitwise identical totals (the replicated
//      parameters never diverge); the SGD update can be applied by that thread in the same kernel.
// There is no grid-wide rendezvous: an element only depends on the same element of the peers, so CTAs do not have to
// be co-resident and a launch can loop over any number of elements (round 1 used a CTA arrival counter + one flag per
// rank, which needed the whole grid resident and cost two NVLink round trips plus a system fence per step).
// Double buffering by `seq & 1` is sufficient: a rank can only write step s+2 (slot s & 1) after it finished step
// s+1, i.e. after every peer pushed step s+1, which a peer does only after its kernel of step s has completed.
#pragma once
#include <stdint.h>

namespace rcmarl {

constexpr int COMM_MAX_WORLD = 8;

struct CommDev {
    uint2* cells[COMM_MAX_WORLD];      // peer base pointers (cell region)
    uint32_t* error;                   // local error word (spin time-out)
    int64_t max_floats;
    int32_t rank, world;
    uint32_t seq;
};

constexpr int CELL_POLL_NS = 40;                           // back-off between polls of a cell that has not arrived yet

__device__ __forceinline__ void st_cell(uint2* p, float v, uint32_t seq) {
    asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(seq) : "memory");
}
__device__ __forceinline__ uint2 ld_cell(const uint2* p) {
    uint2 v;
    asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}

// cell of element `offset` from source rank `src` in slot (seq & 1) of a buffer
__device__ __forceinline__ int64_t comm_index(const CommDev& c, int src, int64_t offset, uint32_t seq) {
    return ((int64_t)(seq & 1u) * c.world + src) * c.max_floats + offset;
}
// step 1: push this rank's value of element `offset` to every peer (own buffer included)
__device__ __forceinline__ void comm_push(const CommDev& c, int64_t offset, float v, uint32_t seq) {
    const int64_t idx = comm_index(c, c.rank, offset, seq);
#pragma unroll
    for (int p = 0; p < COMM_MAX_WORLD; ++p)
        if (p < c.world) st_cell(c.cells[p] + idx, v, seq);
}
// step 2: wait for element `offset` of every rank in OUR buffer, rank-ordered sum
__device__ __forceinline__ float comm_wait_total(const CommDev& c, int64_t offset, uint32_t seq) {
    float v[COMM_MAX_WORLD];
    const long long t0 = clock64();
    const uint2* mine = c.cells[0];
#pragma unroll
    for (int p = 1; p < COMM_MAX_WORLD; ++p) mine = (p == c.rank) ? c.cells[p] : mine;
#pragma unroll
    for (int p = 0; p < COMM_MAX_WORLD; ++p) {
        v[p] = 0.f;
        if (p < c.world) {
            const uint2* cell = mine + comm_index(c, p, offset, seq);
            uint2 x = ld_cell(cell);
            while (x.y != seq) {
                if (clock64() - t0 > 120000000000LL) {   // ~60 s: a peer died; fail loudly instead of hanging the GPU
                    *c.error = 1u;
                    __threadfence_system();
                    __trap();                            // surfaces as a CUDA error at the next synchronisation
                }
                __nanosleep(CELL_POLL_NS);
                x = ld_cell(cell);
            }
            v[p] = __uint_as_float(x.x);
        }
    }
    float tot = 0.f;
#pragma unroll
    for (int p = 0; p < COMM_MAX_WORLD; ++p) tot += v[p];   // rank order: identical bits on every rank
    return tot;
}
__device__ __forceinline__ void comm_push(const CommDev& c, int64_t offset, float v) { comm_push(c, offset, v, c.seq); }
__device__ __forceinline__ float comm_wait_total(const CommDev& c, int64_t offset) { return comm_wait_total(c, offset, c.seq); }

// host side (comm.cu)
struct CommHost;
CommHost* comm_bound();
bool comm_next(CommDev* out, int64_t need_floats);   // fills *out with the next sequence number; false if unbound
bool comm_reserve(CommDev* out, int64_t need_floats, uint32_t count);   // `count` consecutive numbers, out->seq = the first

}  // namespace rcmarl
