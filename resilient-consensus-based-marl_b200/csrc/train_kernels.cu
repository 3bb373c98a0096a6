// train_kernels.cu -- update-round kernels of the RPBCAC hot path (sm_90a, fp32 FFMA).
//
//   values_kernel   K1/K3  batched forward values / TD targets / TD errors / actor probabilities
//   grad_kernel     K2/K7/K9  fused forward + backward of the 20-wide MLPs over a row set (grad_kernel.cuh):
//                   phase 1: two buffer rows per lane, weights broadcast from shared memory;
//                   phase 2: the per-row activation / delta vectors are staged in a warp-private
//                            shared-memory tile and every lane owns one 8x8 tile of the weight-gradient
//                            outer products, accumulated in registers across ALL rows of the CTA;
//                   deterministic two-level reduction (CTA partials -> reduce_kernel).
//   team_kernel     K5+K6  neighbour-head estimates, clipped mean, projection numerators
//   attack_kernel   Byzantine messages crafted per receiver (ALIE / IPM / Gaussian, rcmarl_attack)
//   vector_agg_kernel  distance-based rules over whole messages (Krum, multi-Krum, self-centred clipping, geometric
//                   median; rcmarl_vector_aggregate)
//   dnc_agg_kernel  divide-and-conquer: removes the messages furthest along the top principal direction
//                   (rcmarl_dnc_aggregate)
//   subset_agg_kernel  exact subset selection (MDA, SMEA): averages the n - H messages that agree most as a set
//                   (rcmarl_subset_aggregate)
//   ios_agg_kernel  iterative outlier scissor: drops the message furthest from the re-centred mean H times
//                   (rcmarl_ios_aggregate)
//   nnm_mix_kernel  nearest-neighbour mixing: each message becomes the mean of its n - H nearest (rcmarl_nnm_mix)
//   arc_clip_kernel  adaptive robust clipping: the k_clip messages furthest from the receiver's own are pulled in to
//                   the distance of the next (rcmarl_arc_clip)
//   bucket_mix_kernel  randomized bucketing: the received messages are shuffled into buckets of s and replaced by the
//                   bucket means (rcmarl_bucket_mix)
//   adaptive_attack_kernel  min-max / min-sum Byzantine messages scaled to the receiver's honest spread
//                   (rcmarl_adaptive_attack)
//   tailored_attack_kernel  Byzantine messages tuned against the receiver's own rule and H (rcmarl_tailored_attack)
//   pipeline_attack_kernel  the same search against the receiver's mixing step and rule, DnC included
//                   (rcmarl_pipeline_attack)
//   history_attack_kernel  the same search in the momentum rows of a receiver with momentum, inverted through its
//                   momentum step (rcmarl_history_attack)
//   dissensus_attack_kernel  Byzantine messages that cancel the receiver's honest pull (rcmarl_dissensus_attack)
//   mimic_attack_kernel  copies of the honest message furthest along the tracked principal direction
//                   (rcmarl_mimic_attack)
//   consensus, sgd/adam apply, reward mix: the small glue kernels.
//
// Reference semantics: agents/resilient_CAC_agents.py, agents/adversarial_CAC_agents.py,
// training/train_agents.py:86-163 (cited per entry point in include/rcmarl.h).
#include <algorithm>
#include <cmath>
#include <utility>
#include "common.cuh"
#include "grad_kernel.cuh"
#include "comm.cuh"
#include "minibatch_persist.cuh"

namespace rcmarl {

static thread_local int g_last_cuda = 0;
int last_cuda_error_get() { return g_last_cuda; }
void last_cuda_error_set(int e) { g_last_cuda = e; }

int sm_count_cached() {
    static int n = 0;
    if (n == 0) {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0)
            n = v;
        else
            return 132;  // H100 SXM; not cached so that a later call with a device re-queries
    }
    return n;
}

// ============================================================================================
// values
// ============================================================================================
struct ValuesParams {
    rcmarl_rows rows;
    rcmarl_value_job jobs[RCMARL_MAX_JOBS];
};

// value of R = 2 rows per thread: every broadcast weight quad feeds both rows (see grad_kernel.cuh)
template <int NA, int DIN>
__device__ __forceinline__ void value_term2(const rcmarl_rows& R, const float* sw, int kind, const int64_t (&row)[2],
                                            float (&v)[2]) {
    float x[2][DIN], h1[2][HID], h2[2][HID];
    load_x<NA, DIN>(R, kind, row[0], x[0]);
    load_x<NA, DIN>(R, kind, row[1], x[1]);
    features_rows<DIN, 2>(sw, x, h1, h2);
    v[0] = head1<DIN>(sw, h2[0]);
    v[1] = head1<DIN>(sw, h2[1]);
}

template <int NA>
__global__ void __launch_bounds__(256) values_kernel(const __grid_constant__ ValuesParams P) {
    extern __shared__ __align__(16) float smem[];
    const rcmarl_value_job& job = P.jobs[blockIdx.y];
    const rcmarl_rows& R = P.rows;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n_iter = (R.n_rows + stride - 1) / stride;
    if (job.n_out == NACT) {  // actor.predict: softmax probabilities (single term)
        constexpr int DIN = 2 * NA;
        stage_weights(smem, job.w[0], param_count(DIN, NACT));
        __syncthreads();
        for (int64_t it = 0; it < n_iter; ++it) {
            int64_t m = it * stride + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
            if (m < R.n_rows) {
                int64_t row = row_of(R, m);
                float x[DIN], h1[HID], h2[HID], l[NACT], mx, lse;
                load_x<NA, DIN>(R, job.kind[0], row, x);
                features<DIN>(smem, x, h1, h2);
                head5<DIN>(smem, h2, l);
                if (job.softmax) softmax5(l, mx, lse);
#pragma unroll
                for (int o = 0; o < NACT; ++o) job.out[row * NACT + o] = l[o];
            }
        }
        return;
    }
    for (int t = 0; t < job.n_terms; ++t) {
        const int kind = job.kind[t];
        __syncthreads();
        stage_weights(smem, job.w[t], kind == RCMARL_IN_SA ? param_count(3 * NA, 1) : param_count(2 * NA, 1));
        __syncthreads();
        for (int64_t it = 0; it < n_iter; it += 2) {          // two rows per thread and iteration
            int64_t m[2], row[2];
            bool live[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                m[r] = (it + r) * stride + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
                live[r] = (it + r) < n_iter && m[r] < R.n_rows;
                row[r] = row_of(R, live[r] ? m[r] : 0);
            }
            if (!live[0]) continue;
            float v[2];
            if (kind == RCMARL_IN_SA) value_term2<NA, 3 * NA>(R, smem, kind, row, v);
            else value_term2<NA, 2 * NA>(R, smem, kind, row, v);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if (!live[r]) continue;
                float acc;
                if (t == 0)
                    acc = job.add ? job.add_scale * __ldg(job.add + row[r] * job.add_stride + job.add_off) : 0.f;
                else
                    acc = job.out[row[r]];
                job.out[row[r]] = fmaf(job.scale[t], v[r], acc);
            }
        }
    }
}

// Where the CTA partials of job j live: slots first[j] + y * step, y = 0 .. count[j] - 1, each `stride` floats
// (grad_kernel: consecutive slots of the 1-D grid; team_kernel: [y][job] interleaved).
struct PartialSlots {
    int32_t first[RCMARL_MAX_JOBS];
    int32_t count[RCMARL_MAX_JOBS];
    int32_t step, stride;
};

// Deterministic sum over the CTA partials of one parameter, parallel over the 8 warps of a 256-thread block:
// block b of job j owns parameters [32 b, 32 b + 32); warp w adds y = w, w + 8, ... (coalesced 128-byte rows), the
// eight warp sums are combined in warp order.  Returns the total in the threads of warp 0 (others return 0).
__device__ __forceinline__ float block_partial_sum(const float* __restrict__ partial, const PartialSlots& S, int j, int i,
                                                   bool valid, float* sh /* [8][32] */) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int first = S.first[j], count = S.count[j];
    float s = 0.f;
    if (valid)
        for (int y = warp; y < count; y += 8) s += partial[((int64_t)first + (int64_t)y * S.step) * S.stride + i];
    sh[warp * 32 + lane] = s;
    __syncthreads();
    float tot = 0.f;
    if (warp == 0) {
#pragma unroll
        for (int w = 0; w < 8; ++w) tot += sh[w * 32 + lane];
    }
    return tot;
}

// sums[j][i] = sum_y partial[y][j][i], y ascending (deterministic)
struct ReduceParams {
    const float* partial;
    float* sums[RCMARL_MAX_JOBS];
    int32_t n[RCMARL_MAX_JOBS];
    PartialSlots slots;
};
__global__ void __launch_bounds__(256) reduce_kernel(const __grid_constant__ ReduceParams P) {
    __shared__ float sh[256];
    pdl_launch_dependents();     // the next grad kernel may start its prologue; it waits (pdl_wait) before reading
    const int j = blockIdx.y;
    const int i = blockIdx.x * 32 + (threadIdx.x & 31);
    const bool valid = i < P.n[j];
    const float s = block_partial_sum(P.partial, P.slots, j, i, valid, sh);
    if (threadIdx.x < 32 && valid) P.sums[j][i] = s;
}

// Multi-GPU variant: reduce the CTA partials, exchange over NVLink peer memory (comm.cuh) and write the global sums --
// one kernel, no NCCL call, no host round trip.
struct ReduceCommParams {
    const float* partial;
    float* sums[RCMARL_MAX_JOBS];
    int32_t n[RCMARL_MAX_JOBS];
    PartialSlots slots;
    int32_t out_stride;               // distance between the jobs' blocks in the exchange buffer
    int32_t n_jobs, max_n;            // items = n_jobs x ceil(max_n / 32)
    CommDev comm;
};
__global__ void __launch_bounds__(256) reduce_comm_kernel(const __grid_constant__ ReduceCommParams P) {
    __shared__ float sh[256];
    pdl_launch_dependents();     // the next grad kernel may start its prologue; it waits (pdl_wait) before reading
    pdl_wait();                  // launched as a programmatic dependent of the producer: its partials must be complete
    // One item = 32 consecutive elements of one job.  Items are independent (comm.cuh): a CTA walks its items in
    // ascending order on every rank, so any grid size is deadlock-free and nothing has to be co-resident.
    const int blocks_per_job = (P.max_n + 31) / 32;
    const int n_items = blocks_per_job * P.n_jobs;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int j = item / blocks_per_job;
        const int i = (item - j * blocks_per_job) * 32 + (threadIdx.x & 31);
        const bool valid = i < P.n[j];
        const int64_t off = (int64_t)j * P.out_stride + i;
        const float s = block_partial_sum(P.partial, P.slots, j, i, valid, sh);
        if (threadIdx.x < 32 && valid) {
            comm_push(P.comm, off, s);
            const float tot = comm_wait_total(P.comm, off);
            if (P.sums[j]) P.sums[j][i] = tot;
        }
        __syncthreads();          // sh[] is reused by the next item
    }
}

// ============================================================================================
// team: estimates + clipped mean + projection numerators
// ============================================================================================
struct TeamParams {
    rcmarl_rows rows;
    rcmarl_team_job jobs[RCMARL_MAX_JOBS];
    float* partial;
    int32_t n_jobs;
    int32_t stride;
    // jobs of THIS launch (blockIdx.x -> job index).  rcmarl_team launches the team-reward nets (15 inputs) and the critics
    // (10 inputs) separately: the loop body of one instantiation is ~24 KB of SASS, two of them resident on an SM overflow the
    // instruction cache
    int32_t job_list[RCMARL_MAX_JOBS];
};
constexpr int TEAM_N = HID + 2;  // 20 weights + bias numerators + diagnostic loss

// MAXN: compile-time bound on the neighbour count (4 / 8 / 16) so that the estimate vector and the rank-counting
// order statistics stay in registers without paying for 16 x 16 predicated compares when n_in = 4
template <int NA, int DIN, int MAXN>
__device__ __forceinline__ void team_body(const TeamParams& P, const rcmarl_team_job& job, float* smem) {
    constexpr int NP = param_count(DIN, 1);
    const rcmarl_rows& R = P.rows;
    float* sw = smem;                       // agent's network
    float* heads = smem + round4(NP);       // [n_in][24]: W3 (20), b3, pad
    stage_weights(sw, job.w, NP);
    for (int i = threadIdx.x; i < job.n_in * 24; i += blockDim.x) {
        const int k = i / 24, j = i % 24;
        const float* m = job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride;
        heads[i] = j < HID ? __ldg(m + off_W3(DIN) + j) : (j == HID ? __ldg(m + off_b3(DIN, 1)) : 0.f);
    }
    __syncthreads();
    float acc[TEAM_N];
#pragma unroll
    for (int j = 0; j < TEAM_N; ++j) acc[j] = 0.f;
    const int64_t stride = (int64_t)gridDim.y * blockDim.x;
    const int64_t n_iter = (R.n_rows + stride - 1) / stride;
    for (int64_t it = 0; it < n_iter; it += 2) {                   // two rows per thread and iteration
        int64_t row[2];
        bool live[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int64_t m = (it + r) * stride + (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
            live[r] = (it + r) < n_iter && m < R.n_rows;
            row[r] = row_of(R, live[r] ? m : 0);
        }
        if (!live[0]) continue;
        float phi[2][HID];
        {
            float x[2][DIN], h1[2][HID];
            load_x<NA, DIN>(R, job.kind, row[0], x[0]);
            load_x<NA, DIN>(R, job.kind, row[1], x[1]);
            features_rows<DIN, 2>(sw, x, h1, phi);
        }
        float agg[2];
        if (job.agg_in) {
            agg[0] = __ldg(job.agg_in + row[0]);
            agg[1] = __ldg(job.agg_in + row[1]);
        } else {
            float est[2][MAXN];
#pragma unroll
            for (int k = 0; k < MAXN; ++k) {
                est[0][k] = 0.f;
                est[1][k] = 0.f;
                if (k < job.n_in) {
                    const float* hk = heads + k * 24;
                    float s0 = hk[HID], s1 = hk[HID];
#pragma unroll
                    for (int j = 0; j < HID; ++j) { s0 = fmaf(phi[0][j], hk[j], s0); s1 = fmaf(phi[1][j], hk[j], s1); }
                    est[0][k] = s0;
                    est[1][k] = s1;
                }
            }
            agg[0] = resilient_mean_small<MAXN>(est[0], job.n_in, job.H, job.rule);
            agg[1] = resilient_mean_small<MAXN>(est[1], job.n_in, job.H, job.rule);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!live[r]) continue;
            if (job.agg_out) job.agg_out[row[r]] = agg[r];
            if (job.sums) {
                const float pred = head1<DIN>(sw, phi[r]);
                float nrm = 1.f;
#pragma unroll
                for (int j = 0; j < HID; ++j) nrm = fmaf(phi[r][j], phi[r][j], nrm);
                const float err = agg[r] - pred;
                const float c = err / nrm;
#pragma unroll
                for (int j = 0; j < HID; ++j) acc[j] = fmaf(c, phi[r][j], acc[j]);
                acc[HID] += c;
                acc[HID + 1] = fmaf(err, c, acc[HID + 1]);
            }
        }
    }
    if (!job.sums) return;
    __syncthreads();
    float* red = smem;  // [nwarps][TEAM_N]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
#pragma unroll
    for (int j = 0; j < TEAM_N; ++j) {
        float s = warp_sum(acc[j]);
        if (lane == 0) red[warp * TEAM_N + j] = s;
    }
    __syncthreads();
    if (threadIdx.x < TEAM_N) {
        float s = 0.f;
        for (int w = 0; w < nwarps; ++w) s += red[w * TEAM_N + threadIdx.x];
        P.partial[((int64_t)blockIdx.y * P.n_jobs + P.job_list[blockIdx.x]) * P.stride + threadIdx.x] = s;
    }
}

template <int NA>
__global__ void __launch_bounds__(128) team_kernel(const __grid_constant__ TeamParams P) {
    extern __shared__ __align__(16) float smem[];
    const rcmarl_team_job& job = P.jobs[P.job_list[blockIdx.x]];
    const bool sa = job.kind == RCMARL_IN_SA;
    if (job.n_in <= 4) {
        if (sa) team_body<NA, 3 * NA, 4>(P, job, smem); else team_body<NA, 2 * NA, 4>(P, job, smem);
    } else if (job.n_in <= 8) {
        if (sa) team_body<NA, 3 * NA, 8>(P, job, smem); else team_body<NA, 2 * NA, 8>(P, job, smem);
    } else {
        if (sa) team_body<NA, 3 * NA, 16>(P, job, smem); else team_body<NA, 2 * NA, 16>(P, job, smem);
    }
}

// ============================================================================================
// small kernels
// ============================================================================================
struct ConsensusParams { rcmarl_consensus_job jobs[RCMARL_MAX_JOBS]; };
__global__ void __launch_bounds__(256) consensus_hidden_kernel(const __grid_constant__ ConsensusParams P) {
    const rcmarl_consensus_job& job = P.jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= job.n_hidden) return;
    float v[RCMARL_MAX_NEIGHBOURS];
#pragma unroll
    for (int k = 0; k < RCMARL_MAX_NEIGHBOURS; ++k)
        v[k] = k < job.n_in ? __ldg(job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride + i) : 0.f;
    job.dst[i] = resilient_mean_small<RCMARL_MAX_NEIGHBOURS>(v, job.n_in, job.H, job.rule);
}

// Byzantine messages (rcmarl_attack, include/rcmarl.h): one thread per coordinate; mean and population std over the
// honest set in list order (two passes over registers), then the attack
struct AttackParams { rcmarl_attack_job jobs[RCMARL_MAX_JOBS]; };
__global__ void __launch_bounds__(256) attack_kernel(const __grid_constant__ AttackParams P) {
    const rcmarl_attack_job& job = P.jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= job.n) return;
    const int n = job.n_honest;
    float v[RCMARL_MAX_NEIGHBOURS];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < RCMARL_MAX_NEIGHBOURS; ++k) {
        v[k] = k < n ? __ldg(job.msgs + (int64_t)job.honest[k] * job.msg_stride + i) : 0.f;
        if (k < n) s += v[k];
    }
    const float mu = s / (float)n;
    float m;
    if (job.kind == RCMARL_ATTACK_ALIE) {
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < RCMARL_MAX_NEIGHBOURS; ++k)
            if (k < n) q = fmaf(v[k] - mu, v[k] - mu, q);
        m = mu - job.param * sqrtf(q / (float)n);
    } else if (job.kind == RCMARL_ATTACK_IPM) {
        m = -job.param * mu;
    } else {
        const uint4 r = philox4x32_10(make_uint4((uint32_t)i, job.attacker | job.receiver << 8 | 0x40000000u, job.round,
                                                 job.epoch),
                                      make_uint2((uint32_t)job.seed, (uint32_t)(job.seed >> 32)));
        const float u1 = (float)((r.x >> 8) + 1) * (1.0f / 16777216.0f);
        const float u2 = (float)(r.y >> 8) * (1.0f / 16777216.0f);
        m = mu + job.param * (sqrtf(-2.f * logf(u1)) * cospif(2.f * u2));
    }
    job.dst[i] = m;
}

// Distance-based rules over whole messages (rcmarl_vector_aggregate, include/rcmarl.h): one CTA of 256 threads per job.
// The n_in messages are staged in shared memory; every distance is summed by ONE warp (lane-strided partials, then the
// fixed xor butterfly of warp_sum), so its value does not depend on which warp takes it.  Scores, order statistics and
// weights for n_in <= 16 run on warp 0, one lane per message, on registers and shared memory (no local arrays); the
// output takes one thread per coordinate and adds the messages in index order.
struct VectorParams { rcmarl_vector_job jobs[RCMARL_MAX_JOBS]; };
constexpr int VEC_THREADS = 256;

// squared distance of two shared-memory vectors of n floats, in every lane of the calling warp; not finite -> +inf
__device__ __forceinline__ float warp_sqdist(const float* a, const float* b, int n, int lane) {
    float s = 0.f;
    for (int p = lane; p < n; p += 32) {
        const float d = a[p] - b[p];
        s = fmaf(d, d, s);
    }
    s = warp_sum(s);
    return isfinite(s) ? s : INFINITY;
}

// The messages of a job staged one after another in shared memory: message k at xs + k * n.
struct StagedRows {
    const float* xs;
    int n;
    __device__ __forceinline__ const float* operator()(int k) const { return xs + k * n; }
    __device__ __forceinline__ float at(int k, int p) const { return xs[k * n + p]; }
};

// The body of rcmarl_vector_aggregate over nin messages row(0) .. row(nin - 1) of n floats in shared memory: writes the
// aggregate to out[0:n] and leaves w_k in wt (the caller synchronises before reading either).  z is a shared work row
// of n floats (GMED's iterate) and may be out itself: the last Weiszfeld step reads only the messages and wt.  Shared
// scratch: dist [MAXN * MAXN] (KRUM / MKRUM: D_kl; SCCLIP: d_k in dist[k]), wt [MAXN] (KRUM / MKRUM: w_k; SCCLIP: c_k;
// GMED: beta_k), score [MAXN], total (GMED: sum beta).  Called by the whole CTA of VEC_THREADS threads; Row maps a
// message index to its staged row.
template <class Row>
__device__ __forceinline__ void vector_rule(const Row& row, int n, int nin, int H, int rule, float* z, float* out,
                                            float* dist, float* wt, float* score, float& total) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    constexpr int NW = VEC_THREADS / 32;
    if (rule == RCMARL_VEC_KRUM || rule == RCMARL_VEC_MKRUM) {
        for (int t = warp; t < nin * (nin - 1) / 2; t += NW) {       // unordered pairs k < l
            int k = 0, r = t;
            while (r >= nin - 1 - k) { r -= nin - 1 - k; ++k; }
            const int l = k + 1 + r;
            const float d = warp_sqdist(row(k), row(l), n, lane);
            if (lane == 0) { dist[k * MAXN + l] = d; dist[l * MAXN + k] = d; }
        }
        __syncthreads();
        if (warp == 0) {
            const int k = lane, cnt = nin - H - 2, m = rule == RCMARL_VEC_KRUM ? 1 : nin - H;
            if (k < nin) {
                float v[MAXN];
                int rk[MAXN];
#pragma unroll
                for (int l = 0; l < MAXN; ++l) v[l] = (l < nin && l != k) ? dist[k * MAXN + l] : 0.f;
#pragma unroll
                for (int l = 0; l < MAXN; ++l) {          // rank of D_kl among the l != k, ties to the lower index
                    int r = 0;
#pragma unroll
                    for (int q = 0; q < MAXN; ++q)
                        if (q < nin && q != k) r += (v[q] < v[l] || (v[q] == v[l] && q < l)) ? 1 : 0;
                    rk[l] = (l < nin && l != k) ? r : MAXN;
                }
                float s = 0.f;
#pragma unroll
                for (int q = 0; q < MAXN - 1; ++q) {      // the cnt smallest, in ascending order
                    if (q < cnt) {
#pragma unroll
                        for (int l = 0; l < MAXN; ++l)
                            if (rk[l] == q) s += v[l];
                    }
                }
                score[k] = s;
            }
            __syncwarp();
            if (k < nin) {
                const float sk = score[k];
                int r = 0;
#pragma unroll
                for (int q = 0; q < MAXN; ++q)
                    if (q < nin) r += (score[q] < sk || (score[q] == sk && q < k)) ? 1 : 0;
                wt[k] = r < m ? 1.f / (float)m : 0.f;
            }
        }
        __syncthreads();
        const float fm = rule == RCMARL_VEC_KRUM ? 1.f : (float)(nin - H);
        for (int p = tid; p < n; p += VEC_THREADS) {
            float s = 0.f;
            for (int k = 0; k < nin; ++k)
                if (wt[k] != 0.f) s += row.at(k, p);
            out[p] = s / fm;
        }
    } else if (rule == RCMARL_VEC_SCCLIP) {
        for (int k = 1 + warp; k < nin; k += NW) {
            const float d = sqrtf(warp_sqdist(row(k), row(0), n, lane));
            if (lane == 0) dist[k] = d;
        }
        __syncthreads();
        if (warp == 0) {
            const int k = lane;
            if (k >= 1 && k < nin && H < nin - 1) {       // tau = the d_k of descending rank H (ties to the lower index)
                const float dk = dist[k];
                int r = 0;
                for (int q = 1; q < nin; ++q) r += (dist[q] > dk || (dist[q] == dk && q < k)) ? 1 : 0;
                if (r == H) score[0] = dk;
            }
            __syncwarp();
            const float tau = H < nin - 1 ? score[0] : 0.f;
            if (k >= 1 && k < nin) {
                const float dk = dist[k];
                wt[k] = !isfinite(dk) ? 0.f : (dk <= tau ? 1.f : tau / dk);
            }
        }
        __syncthreads();
        const float fn = (float)nin;
        for (int p = tid; p < n; p += VEC_THREADS) {
            const float x0 = row.at(0, p);
            float s = 0.f;
            for (int k = 1; k < nin; ++k) {
                const float c = wt[k];
                if (c != 0.f) s = fmaf(c, row.at(k, p) - x0, s);
            }
            out[p] = x0 + s / fn;
        }
        __syncthreads();                                              // every c_k read
        if (tid == 0) {
            float sw = 0.f;
            for (int k = 1; k < nin; ++k) {
                wt[k] = wt[k] / fn;
                sw += wt[k];
            }
            wt[0] = 1.f - sw;
        }
    } else {                                                          // GMED
        for (int p = tid; p < n; p += VEC_THREADS) {
            float v[MAXN];
#pragma unroll
            for (int k = 0; k < MAXN; ++k) v[k] = k < nin ? row.at(k, p) : 0.f;
            z[p] = resilient_mean_small<MAXN>(v, nin, (nin - 1) / 2, RCMARL_AGG_TRIM);
        }
        for (int it = 0; it < RCMARL_GMED_ITERS; ++it) {
            __syncthreads();                                          // z complete
            for (int k = warp; k < nin; k += NW) {
                const float d = sqrtf(warp_sqdist(row(k), z, n, lane));
                if (lane == 0) wt[k] = isfinite(d) ? 1.f / fmaxf(d, RCMARL_GMED_NU) : 0.f;
            }
            __syncthreads();
            if (tid == 0) {
                float s = 0.f;
                for (int k = 0; k < nin; ++k) s += wt[k];
                if (s == 0.f) { wt[0] = 1.f; s = 1.f; }               // no finite distance: out = x_0
                total = s;
            }
            __syncthreads();
            const float St = total;
            float* o = it == RCMARL_GMED_ITERS - 1 ? out : z;
            for (int p = tid; p < n; p += VEC_THREADS) {
                float s = 0.f;
                for (int k = 0; k < nin; ++k) {
                    const float b = wt[k];
                    if (b != 0.f) s = fmaf(b, row.at(k, p), s);
                }
                o[p] = s / St;
            }
        }
        __syncthreads();                                              // every beta_k read
        if (tid == 0)
            for (int k = 0; k < nin; ++k) wt[k] = wt[k] / total;
    }
}

__global__ void __launch_bounds__(VEC_THREADS) vector_agg_kernel(const __grid_constant__ VectorParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    extern __shared__ __align__(16) float smem[];
    __shared__ float dist[MAXN * MAXN];
    __shared__ float wt[MAXN];
    __shared__ float score[MAXN];
    __shared__ float total;
    const rcmarl_vector_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    float* xs = smem;                              // [n_in][n]
    float* z = smem + (int64_t)nin * n;            // GMED iterate [n]
    for (int k = 0; k < nin; ++k) {
        const float* src = job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride;
        for (int p = tid; p < n; p += VEC_THREADS) xs[k * n + p] = __ldg(src + p);
    }
    __syncthreads();
    vector_rule(StagedRows{xs, n}, n, nin, job.H, job.rule, z, job.dst, dist, wt, score, total);
    if (job.weights_out) {
        __syncthreads();
        if (tid < nin) job.weights_out[tid] = wt[tid];
    }
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Cyclic Jacobi on the symmetric m x m fp64 matrix A (m <= RCMARL_MAX_NEIGHBOURS, row stride RCMARL_MAX_NEIGHBOURS) in
// shared memory, run by the calling warp, lane k owning row k, every lane computing each rotation identically: pairs
// p < q in row order; a rotation is skipped, and A_pq set to 0, when 100 |A_pq| is below the rounding of |A_pp| and of
// |A_qq|; at most RCMARL_DNC_SWEEPS sweeps, ending early after a sweep without a rotation.  The eigenvalues are left on
// the diagonal.  V, when not null, is set to the identity and accumulates the rotations: column c is the eigenvector
// of A_cc.  The rule of include/rcmarl.h for DnC's and SMEA's eigen-solves.
__device__ __forceinline__ void warp_jacobi(double* A, double* V, int m) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    const int k = threadIdx.x & 31;
    if (V && k < m)
        for (int c = 0; c < m; ++c) V[k * MAXN + c] = c == k ? 1.0 : 0.0;
    __syncwarp();
    for (int sweep = 0; sweep < RCMARL_DNC_SWEEPS; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < m - 1; ++p) {
            for (int q = p + 1; q < m; ++q) {
                const double apq = A[p * MAXN + q], app = A[p * MAXN + p], aqq = A[q * MAXN + q];
                const double g = 100.0 * fabs(apq);
                __syncwarp();                                       // every lane has read them
                if (apq == 0.0 || (fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq))) {
                    if (k == 0) { A[p * MAXN + q] = 0.0; A[q * MAXN + p] = 0.0; }
                    __syncwarp();
                    continue;
                }
                rotated = true;
                const double theta = (aqq - app) / (2.0 * apq);
                const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + hypot(theta, 1.0));
                const double c = 1.0 / sqrt(fma(tt, tt, 1.0)), s = tt * c;
                if (k < m && k != p && k != q) {
                    const double akp = A[k * MAXN + p], akq = A[k * MAXN + q];
                    const double nkp = c * akp - s * akq, nkq = s * akp + c * akq;
                    A[k * MAXN + p] = nkp; A[p * MAXN + k] = nkp;
                    A[k * MAXN + q] = nkq; A[q * MAXN + k] = nkq;
                } else if (k == p) {
                    A[p * MAXN + p] = app - tt * apq;
                    A[q * MAXN + q] = aqq + tt * apq;
                    A[p * MAXN + q] = 0.0; A[q * MAXN + p] = 0.0;
                }
                if (V && k < m) {
                    const double vkp = V[k * MAXN + p], vkq = V[k * MAXN + q];
                    V[k * MAXN + p] = c * vkp - s * vkq;
                    V[k * MAXN + q] = s * vkp + c * vkq;
                }
                __syncwarp();
            }
        }
        if (!rotated) break;
    }
}

// Divide-and-conquer (rcmarl_dnc_aggregate, include/rcmarl.h): one CTA of VEC_THREADS threads per job.  The fp32
// messages and the fp64 mean of the unflagged ones are staged in shared memory; every Gram entry is summed by ONE warp
// (lane-strided fp64 fma partials, then the fixed xor butterfly), so its value does not depend on which warp takes it.
// The Jacobi eigen-solve runs on warp 0, one lane per row of the m x m matrix, with every lane computing each rotation
// identically; scores, selection and weights also run on warp 0, and the output takes one thread per coordinate.
struct DncShared {
    double A[RCMARL_MAX_NEIGHBOURS * RCMARL_MAX_NEIGHBOURS];   // G, reduced in place by the Jacobi rotations
    double V[RCMARL_MAX_NEIGHBOURS * RCMARL_MAX_NEIGHBOURS];   // the accumulated rotations: column c is the eigenvector of A[c][c]
    int ulist[RCMARL_MAX_NEIGHBOURS];                          // U in index order
    int flagged[RCMARL_MAX_NEIGHBOURS];
    float wt[RCMARL_MAX_NEIGHBOURS];
    int m;
};

// The body of rcmarl_dnc_aggregate over nin messages row(0) .. row(nin - 1) of n floats in shared memory: writes the
// aggregate to out[0:n] and leaves w_k in S.wt (the caller synchronises before reading either).  mu is a shared work
// row of n doubles.  Called by the whole CTA of VEC_THREADS threads; Row maps a message index to its staged row.
template <class Row>
__device__ __forceinline__ void dnc_rule(const Row& row, int n, int nin, int H, double* mu, float* out, DncShared& S) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr int NW = VEC_THREADS / 32;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    double* A = S.A;
    double* V = S.V;
    for (int k = warp; k < nin; k += NW) {
        bool inf = false;
        for (int p = lane; p < n; p += 32) inf |= isinf(row.at(k, p));
        inf = __any_sync(0xffffffffu, inf);
        if (lane == 0) S.flagged[k] = inf ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) {
        int m = 0;
        for (int k = 0; k < nin; ++k)
            if (!S.flagged[k]) S.ulist[m++] = k;
        S.m = m;
    }
    __syncthreads();
    const int m = S.m;
    if (m > 0) {
        const double inv_m = 1.0 / (double)m;
        for (int p = tid; p < n; p += VEC_THREADS) {
            double s = 0.0;
            for (int a = 0; a < m; ++a) s += (double)row.at(S.ulist[a], p);
            mu[p] = s * inv_m;
        }
        __syncthreads();
        for (int t = warp; t < m * (m + 1) / 2; t += NW) {          // pairs a <= b of U positions
            int a = 0, r = t;
            while (r >= m - a) { r -= m - a; ++a; }
            const int b = a + r;
            const float* xa = row(S.ulist[a]);
            const float* xb = row(S.ulist[b]);
            double s = 0.0;
            for (int p = lane; p < n; p += 32) s = fma((double)xa[p] - mu[p], (double)xb[p] - mu[p], s);
            s = warp_sum_f64(s);
            if (lane == 0) { A[a * MAXN + b] = s; A[b * MAXN + a] = s; }
        }
        __syncthreads();
        if (warp == 0) {
            const int k = lane;
            warp_jacobi(A, V, m);
            // lambda = the largest diagonal entry (ties to the lower index), score of U position a = lambda * u_a^2
            int top = 0;
            for (int c = 1; c < m; ++c)
                if (A[c * MAXN + c] > A[top * MAXN + top]) top = c;
            const double lambda = A[top * MAXN + top];
            // U position of lane k's row (k < nin), or -1 if flagged; its score
            int pos = -1;
            for (int a = 0; a < m; ++a)
                if (S.ulist[a] == k) pos = a;
            double sc = INFINITY;
            if (pos >= 0) {
                const double u = V[pos * MAXN + top];
                sc = lambda * (u * u);
            }
            // rows above k in the removal order: a higher score, or an equal one at a higher index (F is all +inf)
            const int n_flag = nin - m, n_rm = max(n_flag, H);
            int above = 0;
            for (int l = 0; l < nin; ++l) {
                const double sl = __shfl_sync(0xffffffffu, sc, l);
                if (l != k && l < nin) above += (sl > sc || (sl == sc && l > k)) ? 1 : 0;
            }
            if (k < nin) S.wt[k] = above < n_rm ? 0.f : 1.f / (float)(nin - n_rm);
        }
    } else if (tid < nin) {
        S.wt[tid] = tid == 0 ? 1.f : 0.f;                            // every row flagged: out = x_0
    }
    __syncthreads();
    for (int p = tid; p < n; p += VEC_THREADS) {                     // cnt = |I| (1 when every row is flagged)
        float s = 0.f, cnt = 0.f;
        for (int k = 0; k < nin; ++k)
            if (S.wt[k] != 0.f) { s += row.at(k, p); cnt += 1.f; }
        out[p] = s / cnt;
    }
}

__global__ void __launch_bounds__(VEC_THREADS) dnc_agg_kernel(const __grid_constant__ VectorParams P) {
    extern __shared__ __align__(16) float smem[];
    __shared__ DncShared S;
    const rcmarl_vector_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    double* mu = reinterpret_cast<double*>(smem);  // [n]
    float* xs = smem + 2 * (int64_t)n;             // [n_in][n]
    for (int k = 0; k < nin; ++k) {
        const float* src = job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride;
        for (int p = tid; p < n; p += VEC_THREADS) xs[k * n + p] = __ldg(src + p);
    }
    __syncthreads();
    dnc_rule(StagedRows{xs, n}, n, nin, job.H, mu, job.dst, S);
    if (job.weights_out && tid < nin) job.weights_out[tid] = S.wt[tid];
}

// Exact subset selection (rcmarl_subset_aggregate, include/rcmarl.h): one CTA of VEC_THREADS threads per job.  The
// messages are staged in shared memory, rows holding +-inf are flagged as in dnc_rule, and every fp64 distance of a
// pair of U positions is summed by ONE warp (lane-strided fma partials, then the fixed xor butterfly).  A candidate is
// a bit mask over U positions; rank r is unranked by the combinatorial number system, so the walk below visits ranks in
// a fixed order whatever the data.  MDA takes one thread per candidate (ranks tid, tid + VEC_THREADS, ...); SMEA one
// warp per candidate (ranks warp, warp + NW, ...), lane a owning row a of B_S in the warp's own scratch, solved by
// warp_jacobi without eigenvectors.  Each thread keeps its best (c, rank), the earlier rank on equal c; warp 0 then
// reduces them to S* by the order (c, rank), and the output takes one thread per coordinate.
struct SubsetShared {
    double D[RCMARL_MAX_NEIGHBOURS * RCMARL_MAX_NEIGHBOURS];                      // D over U positions, D_aa = 0
    double B[VEC_THREADS / 32][RCMARL_MAX_NEIGHBOURS * RCMARL_MAX_NEIGHBOURS];    // SMEA: B_S of each warp's candidate
    double best_c[VEC_THREADS];
    int best_r[VEC_THREADS];
    int binom[RCMARL_MAX_NEIGHBOURS + 1][RCMARL_MAX_NEIGHBOURS + 1];             // C(a, b), 0 for b > a
    int ulist[RCMARL_MAX_NEIGHBOURS];                                             // U in index order
    int flagged[RCMARL_MAX_NEIGHBOURS];
    float wt[RCMARL_MAX_NEIGHBOURS];
    int m;
};

// The candidate of lexicographic rank r among the sz-subsets of m U positions, as a bit mask (bit a: position a).
__device__ __forceinline__ unsigned subset_unrank(int r, int m, int sz, const int (*binom)[RCMARL_MAX_NEIGHBOURS + 1]) {
    unsigned mask = 0u;
    int a = 0;
    for (int i = 0; i < sz; ++i) {
        for (;;) {                                  // the subsets whose i-th element is a and that share the first i
            const int c = binom[m - 1 - a][sz - 1 - i];
            if (r < c) break;
            r -= c;
            ++a;
        }
        mask |= 1u << a;
        ++a;
    }
    return mask;
}

// C(a, b) for a, b <= RCMARL_MAX_NEIGHBOURS into S.binom; called by the whole CTA, the caller synchronises.
__device__ __forceinline__ void subset_binom(SubsetShared& S) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    for (int e = threadIdx.x; e < (MAXN + 1) * (MAXN + 1); e += VEC_THREADS) {
        const int a = e / (MAXN + 1), b = e % (MAXN + 1);
        int c = b > a ? 0 : 1;
        for (int i = 0; i < b && i < a; ++i) c = c * (a - i) / (i + 1);
        S.binom[a][b] = c;
    }
}

// Whether row xa holds +-inf, in every lane of the calling warp (the flag of rcmarl_subset_aggregate and dnc_rule).
__device__ __forceinline__ bool warp_has_inf(const float* xa, int n, int lane) {
    bool inf = false;
    for (int p = lane; p < n; p += 32) inf |= isinf(xa[p]);
    return __any_sync(0xffffffffu, inf);
}

// The fp64 squared distance of two rows in every lane of the calling warp: lane-strided fma partials, then the fixed
// xor butterfly (rcmarl_subset_aggregate's D_kl).
__device__ __forceinline__ double warp_sqdist_f64(const float* xa, const float* xb, int n, int lane) {
    double s = 0.0;
    for (int p = lane; p < n; p += 32) {
        const double d = (double)xa[p] - (double)xb[p];
        s = fma(d, d, s);
    }
    return warp_sum_f64(s);
}

// The argmin over (c, rank), a total order, of (bc, br) of the calling lane and S.best_c / S.best_r of every thread
// past warp 0, into (bc, br) of every lane of warp 0.
__device__ __forceinline__ void subset_argmin(const SubsetShared& S, double& bc, int& br, int lane) {
    for (int q = lane + 32; q < VEC_THREADS; q += 32) {
        const double c = S.best_c[q];
        const int r = S.best_r[q];
        if (c < bc || (c == bc && r < br)) { bc = c; br = r; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const double c = __shfl_xor_sync(0xffffffffu, bc, o);
        const int r = __shfl_xor_sync(0xffffffffu, br, o);
        if (c < bc || (c == bc && r < br)) { bc = c; br = r; }
    }
}

// The rows of `known` whose flags and pairwise distances subset_rule reads from a cache instead of its rows: flag[k]
// for k in known, DK[k * MAXN + l] (row indices) for k != l both in known and unflagged.  Called by the whole CTA; the
// caller synchronises.
template <class Row>
__device__ __forceinline__ void subset_known(const Row& row, int n, int nin, unsigned known, int* flag, double* DK) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr int NW = VEC_THREADS / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int k = warp; k < nin; k += NW)
        if ((known >> k) & 1u) {
            const bool inf = warp_has_inf(row(k), n, lane);
            if (lane == 0) flag[k] = inf ? 1 : 0;
        }
    __syncthreads();
    for (int t = warp; t < nin * nin; t += NW) {
        const int k = t / nin, l = t % nin;
        if (k < l && ((known >> k) & (known >> l) & 1u) && !flag[k] && !flag[l]) {
            const double s = warp_sqdist_f64(row(k), row(l), n, lane);
            if (lane == 0) { DK[k * MAXN + l] = s; DK[l * MAXN + k] = s; }
        }
    }
}

// The best (criterion, rank) over the candidates that hold only rows of `known`, for the U (as a row mask) it was
// taken with; urows = 0 until it is taken.
struct SubsetKnownBest {
    double c;
    int r;
    unsigned urows;
};

// The body of rcmarl_subset_aggregate over nin rows row(0) .. row(nin - 1) of n floats in shared memory (S.binom
// filled): writes the aggregate to out[0:n] and leaves w_k in S.wt (the caller synchronises before reading either).
// The rows of `known` take their flags from kflag and the distances of their pairs from DK (subset_known, the same
// warp code), so only the pairs with a row outside `known` are summed here.  With kb, the candidates that hold only
// rows of `known` are searched once: the first call takes their best (c, rank) into kb besides the full search, and a
// later call with the same U skips them and merges kb's -- the same criteria from the same numbers, and (c, rank) is a
// total order, so the selection is the full search's.  Called by the whole CTA of VEC_THREADS threads; Row maps a row
// index to its staged row.
template <class Row>
__device__ __forceinline__ void subset_rule(const Row& row, int n, int nin, int H, int rule, float* out, SubsetShared& S,
                                            unsigned known = 0u, const int* kflag = nullptr,
                                            const double* DK = nullptr, SubsetKnownBest* kb = nullptr) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr int NW = VEC_THREADS / 32;
    const bool smea = rule == RCMARL_SUBSET_SMEA;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int k = warp; k < nin; k += NW) {
        if ((known >> k) & 1u) {
            if (lane == 0) S.flagged[k] = kflag[k];
            continue;
        }
        const bool inf = warp_has_inf(row(k), n, lane);
        if (lane == 0) S.flagged[k] = inf ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) {
        int m = 0;
        for (int k = 0; k < nin; ++k)
            if (!S.flagged[k]) S.ulist[m++] = k;
        S.m = m;
    }
    __syncthreads();
    const int m = S.m;
    if (m > 0) {
        for (int t = warp; t < m * (m - 1) / 2; t += NW) {          // pairs a < b of U positions
            int a = 0, r = t;
            while (r >= m - 1 - a) { r -= m - 1 - a; ++a; }
            const int b = a + 1 + r;
            const int ia = S.ulist[a], ib = S.ulist[b];
            const double s = ((known >> ia) & (known >> ib) & 1u) ? DK[ia * MAXN + ib]
                                                                   : warp_sqdist_f64(row(ia), row(ib), n, lane);
            if (lane == 0) { S.D[a * MAXN + b] = s; S.D[b * MAXN + a] = s; }
        }
        if (tid < m) S.D[tid * MAXN + tid] = 0.0;
        __syncthreads();
        const int sz = nin - max(nin - m, H);                        // >= 1
        const int total = S.binom[m][sz];
        double bc = INFINITY, kc = INFINITY;
        int br = 0x7fffffff, kr = 0x7fffffff;
        unsigned urows = 0u, kpos = 0u;                               // kb: U as a row mask, the known U positions
        if (kb)
            for (int a = 0; a < m; ++a) {
                urows |= 1u << S.ulist[a];
                kpos |= ((known >> S.ulist[a]) & 1u) << a;
            }
        const bool use = kb && sz > 1 && kb->urows == urows;          // skip the known-only candidates, merge kb's
        const bool take = kb && sz > 1 && kb->urows == 0u;            // and take kb in this call
        if (sz == 1) {                                                // every criterion is 0: rank 0
            bc = 0.0;
            br = 0;
        } else if (!smea) {
            for (int r = tid; r < total; r += VEC_THREADS) {
                const unsigned mask = subset_unrank(r, m, sz, S.binom);
                const bool konly = (mask & ~kpos) == 0u;
                if (use && konly) continue;
                double c = 0.0;
                for (unsigned ma = mask; ma; ma &= ma - 1) {
                    const int a = __ffs(ma) - 1;
                    for (unsigned mb = ma & (ma - 1); mb; mb &= mb - 1) {
                        const double d = S.D[a * MAXN + __ffs(mb) - 1];
                        if (d > c) c = d;
                    }
                }
                if (c < bc) { bc = c; br = r; }
                if (take && konly && c < kc) { kc = c; kr = r; }
            }
        } else {
            double* B = S.B[warp];
            for (int r = warp; r < total; r += NW) {
                const unsigned mask = subset_unrank(r, m, sz, S.binom);
                const bool konly = (mask & ~kpos) == 0u;              // the same in every lane
                if (use && konly) continue;
                int pa = 0;                                           // lane a < sz: the a-th position of the subset
                unsigned mm = mask;
                for (int i = 0; i < lane && mm; ++i) mm &= mm - 1;
                if (mm) pa = __ffs(mm) - 1;
                double ra = 0.0;                                      // r_a = (sum_b D_ab, b in order) / s
                for (int b = 0; b < sz; ++b) {
                    const int pb = __shfl_sync(0xffffffffu, pa, b);
                    if (lane < sz) ra += S.D[pa * MAXN + pb];
                }
                ra = ra / (double)sz;
                double t = 0.0;                                       // t = (sum_a r_a, a in order) / s
                for (int b = 0; b < sz; ++b) t += __shfl_sync(0xffffffffu, ra, b);
                t = t / (double)sz;
                for (int b = 0; b < sz; ++b) {                        // B_ab for a <= b, mirrored
                    const int pb = __shfl_sync(0xffffffffu, pa, b);
                    const double rb = __shfl_sync(0xffffffffu, ra, b);
                    if (lane <= b) {
                        const double v = -0.5 * (((S.D[pa * MAXN + pb] - ra) - rb) + t);
                        B[lane * MAXN + b] = v;
                        B[b * MAXN + lane] = v;
                    }
                }
                __syncwarp();
                warp_jacobi(B, nullptr, sz);
                double c = B[0];
                for (int a = 1; a < sz; ++a) c = fmax(c, B[a * MAXN + a]);
                __syncwarp();                                         // every lane has read the diagonal
                if (c < bc) { bc = c; br = r; }
                if (take && konly && c < kc) { kc = c; kr = r; }
            }
        }
        S.best_c[tid] = bc;
        S.best_r[tid] = br;
        __syncthreads();
        if (warp == 0) {
            subset_argmin(S, bc, br, lane);
            if (use && (kb->c < bc || (kb->c == bc && kb->r < br))) { bc = kb->c; br = kb->r; }
            const unsigned mask = subset_unrank(br, m, sz, S.binom);
            if (lane < nin) S.wt[lane] = 0.f;
            __syncwarp();
            if (lane < m && ((mask >> lane) & 1u)) S.wt[S.ulist[lane]] = 1.f / (float)sz;
        }
        if (take) {                                                   // the same in every thread
            __syncthreads();                                          // warp 0 has read every best
            S.best_c[tid] = kc;
            S.best_r[tid] = kr;
            __syncthreads();
            if (warp == 0) {
                subset_argmin(S, kc, kr, lane);
                if (lane == 0) { kb->c = kc; kb->r = kr; kb->urows = urows; }
            }
        }
    } else if (tid < nin) {
        S.wt[tid] = tid == 0 ? 1.f : 0.f;                            // every row flagged: out = x_0
    }
    __syncthreads();
    for (int p = tid; p < n; p += VEC_THREADS) {                     // cnt = s (1 when every row is flagged)
        float s = 0.f, cnt = 0.f;
        for (int k = 0; k < nin; ++k)
            if (S.wt[k] != 0.f) { s += row.at(k, p); cnt += 1.f; }
        out[p] = s / cnt;
    }
}

__global__ void __launch_bounds__(VEC_THREADS) subset_agg_kernel(const __grid_constant__ VectorParams P) {
    extern __shared__ __align__(16) float smem[];
    __shared__ SubsetShared S;
    const rcmarl_vector_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    float* xs = smem;                              // [n_in][n]
    for (int k = 0; k < nin; ++k) {
        const float* src = job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride;
        for (int p = tid; p < n; p += VEC_THREADS) xs[k * n + p] = __ldg(src + p);
    }
    subset_binom(S);
    __syncthreads();
    subset_rule(StagedRows{xs, n}, n, nin, job.H, job.rule, job.dst, S);
    if (job.weights_out && tid < nin) job.weights_out[tid] = S.wt[tid];
}

// Iterative outlier scissor (rcmarl_ios_aggregate, include/rcmarl.h): one CTA of VEC_THREADS threads per job.  The
// fp32 messages and the fp64 centre are staged in shared memory, rows holding +-inf are flagged as in dnc_rule, and the
// rows still held are a bit mask.  Each iteration recomputes the centre from scratch (one thread per coordinate, rows
// in index order) and sums each d_k on ONE warp (lane-strided fma partials, then the fixed xor butterfly), so no value
// depends on which warp takes a row; thread 0 then removes the argmax, scanning upwards with >= so that equal
// distances remove the higher index.  The output takes one thread per coordinate, as in dnc_rule.
struct IosShared {
    double d[RCMARL_MAX_NEIGHBOURS];
    int flagged[RCMARL_MAX_NEIGHBOURS];
    float wt[RCMARL_MAX_NEIGHBOURS];
    unsigned held;
    int iters;
};

// The body of rcmarl_ios_aggregate over nin rows row(0) .. row(nin - 1) of n floats in shared memory: writes the
// aggregate to out[0:n] and leaves w_k in S.wt (the caller synchronises before reading either).  c is a shared work
// row of n doubles (the centre).  Called by the whole CTA of VEC_THREADS threads; Row maps a row index to its staged
// row.
template <class Row>
__device__ __forceinline__ void ios_rule(const Row& row, int n, int nin, int H, double* c, float* out, IosShared& S) {
    constexpr int NW = VEC_THREADS / 32;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int k = warp; k < nin; k += NW) {
        const bool inf = warp_has_inf(row(k), n, lane);
        if (lane == 0) S.flagged[k] = inf ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) {
        unsigned u = 0u;
        int nf = 0;
        for (int k = 0; k < nin; ++k) {
            if (S.flagged[k]) ++nf;
            else u |= 1u << k;
        }
        S.held = u;
        S.iters = u ? max(0, H - nf) : 0;
    }
    __syncthreads();
    const int n_iter = S.iters;
    for (int it = 0; it < n_iter; ++it) {
        const unsigned u = S.held;
        const double m = (double)__popc(u);
        for (int p = tid; p < n; p += VEC_THREADS) {
            double s = 0.0;
            for (unsigned r = u; r; r &= r - 1) s += (double)row.at(__ffs(r) - 1, p);
            c[p] = s / m;
        }
        __syncthreads();
        for (int k = warp; k < nin; k += NW) {
            if (!((u >> k) & 1u)) continue;
            const float* xk = row(k);
            double s = 0.0;
            for (int p = lane; p < n; p += 32) {
                const double e = (double)xk[p] - c[p];
                s = fma(e, e, s);
            }
            s = warp_sum_f64(s);
            if (lane == 0) S.d[k] = s;
        }
        __syncthreads();
        if (tid == 0) {
            int top = -1;
            for (unsigned r = u; r; r &= r - 1) {
                const int k = __ffs(r) - 1;
                if (top < 0 || S.d[k] >= S.d[top]) top = k;
            }
            S.held = u & ~(1u << top);
        }
        __syncthreads();
    }
    if (tid < nin) {
        const unsigned u = S.held ? S.held : 1u;                     // every row flagged: out = x_0
        S.wt[tid] = ((u >> tid) & 1u) ? 1.f / (float)__popc(u) : 0.f;
    }
    __syncthreads();
    for (int p = tid; p < n; p += VEC_THREADS) {                     // cnt = |I| (1 when every row is flagged)
        float s = 0.f, cnt = 0.f;
        for (int k = 0; k < nin; ++k)
            if (S.wt[k] != 0.f) { s += row.at(k, p); cnt += 1.f; }
        out[p] = s / cnt;
    }
}

__global__ void __launch_bounds__(VEC_THREADS) ios_agg_kernel(const __grid_constant__ VectorParams P) {
    extern __shared__ __align__(16) float smem[];
    __shared__ IosShared S;
    const rcmarl_vector_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    double* c = reinterpret_cast<double*>(smem);   // [n]
    float* xs = smem + 2 * (int64_t)n;             // [n_in][n]
    for (int k = 0; k < nin; ++k) {
        const float* src = job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride;
        for (int p = tid; p < n; p += VEC_THREADS) xs[k * n + p] = __ldg(src + p);
    }
    __syncthreads();
    ios_rule(StagedRows{xs, n}, n, nin, job.H, c, job.dst, S);
    if (job.weights_out && tid < nin) job.weights_out[tid] = S.wt[tid];
}

// Nearest-neighbour mixing (rcmarl_nnm_mix, include/rcmarl.h): one CTA of VEC_THREADS threads per job.  The n_in
// messages are staged in shared memory and every distance of a pair k < l is summed by ONE warp with warp_sqdist, as in
// vector_rule, so D_kl is bitwise Krum's.  The selections N_k run on warp 0, one lane per k, with rank counts over
// registers, and are kept as bit masks; the output takes one thread per coordinate and adds each N_k in index order.
//
// The body over nin messages row(0) .. row(nin - 1) of n floats in shared memory: writes mixed row k to dst(k)[0:n] and
// leaves N_k in sel[k] (bit l set for l in N_k).  Shared scratch: dist [MAXN * MAXN].  Called by the whole CTA of
// VEC_THREADS threads; the caller synchronises before reading a mixed row.
template <class Row, class Dst>
__device__ __forceinline__ void nnm_rows(const Row& row, int n, int nin, int H, float* dist, unsigned* sel,
                                         const Dst& dst) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr int NW = VEC_THREADS / 32;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int t = warp; t < nin * (nin - 1) / 2; t += NW) {           // unordered pairs k < l
        int k = 0, r = t;
        while (r >= nin - 1 - k) { r -= nin - 1 - k; ++k; }
        const int l = k + 1 + r;
        const float d = warp_sqdist(row(k), row(l), n, lane);
        if (lane == 0) { dist[k * MAXN + l] = d; dist[l * MAXN + k] = d; }
    }
    __syncthreads();
    if (warp == 0 && lane < nin) {
        const int k = lane, m = nin - H;
        float v[MAXN];
#pragma unroll
        for (int l = 0; l < MAXN; ++l) v[l] = (l < nin && l != k) ? dist[k * MAXN + l] : 0.f;
        unsigned mask = 0u;
#pragma unroll
        for (int l = 0; l < MAXN; ++l) {              // rank of l in the order (D_kl, l != k, l)
            int r = 0;
#pragma unroll
            for (int q = 0; q < MAXN; ++q)
                if (q < nin && q != l) r += (v[q] < v[l] || (v[q] == v[l] && (q == k || (l != k && q < l)))) ? 1 : 0;
            if (l < nin && r < m && v[l] < INFINITY) mask |= 1u << l;
        }
        sel[k] = mask;
    }
    __syncthreads();
    for (int k = 0; k < nin; ++k) {
        const unsigned mask = sel[k];
        const float cnt = (float)__popc(mask);
        float* out = dst(k);
        for (int p = tid; p < n; p += VEC_THREADS) {
            float s = 0.f;
            for (int l = 0; l < nin; ++l)
                if ((mask >> l) & 1u) s += row.at(l, p);
            out[p] = s / cnt;
        }
    }
}

__global__ void __launch_bounds__(VEC_THREADS) nnm_mix_kernel(const __grid_constant__ VectorParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    static_assert(MAXN * MAXN <= VEC_THREADS, "one thread per entry of M");
    extern __shared__ __align__(16) float smem[];
    __shared__ float dist[MAXN * MAXN];
    __shared__ unsigned sel[MAXN];                 // N_k: bit l set for l in N_k
    const rcmarl_vector_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    float* xs = smem;                              // [n_in][n]
    for (int k = 0; k < nin; ++k) {
        const float* src = job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride;
        for (int p = tid; p < n; p += VEC_THREADS) xs[k * n + p] = __ldg(src + p);
    }
    __syncthreads();
    nnm_rows(StagedRows{xs, n}, n, nin, job.H, dist, sel,
             [&](int k) { return job.dst + (int64_t)k * job.msg_stride; });
    if (job.weights_out && tid < nin * nin) {
        const unsigned mask = sel[tid / nin];
        job.weights_out[tid] = ((mask >> (tid % nin)) & 1u) ? 1.f / (float)__popc(mask) : 0.f;
    }
}

// ARC's factors (rcmarl_arc_clip, include/rcmarl.h) on one warp, lane k for slot k: tau = the d_k (dist[1 .. nin - 1])
// of descending rank k_clip, ties to the lower index (0 if k_clip >= nin - 1), then cf[k] for k < nin.  tau_at is shared
// scratch.  Shared by arc_clip_kernel and the ARC forms of the pipeline and history searches.
__device__ __forceinline__ void arc_factors(const float* dist, int nin, int H, float& tau_at, float* cf, int lane) {
    const int k = lane, kc = 2 * H * (nin - H) / nin;
    if (k >= 1 && k < nin && kc < nin - 1) {
        const float dk = dist[k];
        int r = 0;
        for (int q = 1; q < nin; ++q) r += (dist[q] > dk || (dist[q] == dk && q < k)) ? 1 : 0;
        if (r == kc) tau_at = dk;
    }
    __syncwarp();
    const float tau = kc < nin - 1 ? tau_at : 0.f;
    if (k < nin) {
        const float dk = k == 0 ? 0.f : dist[k];
        cf[k] = !isfinite(dk) ? 0.f : (dk <= tau ? 1.f : __fdiv_rn(tau, dk));
    }
}

// Adaptive robust clipping (rcmarl_arc_clip, include/rcmarl.h): one CTA of VEC_THREADS threads per job.  Nothing is
// staged: each d_k is summed by ONE warp with warp_sqdist straight from global memory, in the order scclip's d_k takes
// in vector_rule, so the two are bitwise equal.  tau and the factors run on warp 0, one lane per slot; the rows take one
// thread per coordinate, every operation rounded on its own (no FMA).
__global__ void __launch_bounds__(VEC_THREADS) arc_clip_kernel(const __grid_constant__ VectorParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr int NW = VEC_THREADS / 32;
    __shared__ float dist[MAXN];
    __shared__ float cf[MAXN];
    __shared__ float tau_at;
    const rcmarl_vector_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    auto row = [&](int k) { return job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride; };
    const float* x0 = row(0);
    for (int k = 1 + warp; k < nin; k += NW) {
        const float d = sqrtf(warp_sqdist(row(k), x0, n, lane));
        if (lane == 0) dist[k] = d;
    }
    __syncthreads();
    if (warp == 0) arc_factors(dist, nin, job.H, tau_at, cf, lane);
    __syncthreads();
    for (int k = 0; k < nin; ++k) {
        const float c = cf[k];
        const float* xk = row(k);
        float* out = job.dst + (int64_t)k * job.msg_stride;
        if (c == 1.f || c == 0.f) {                   // a bitwise copy of x_k or x_0: one row read
            const float* src = c == 1.f ? xk : x0;
            for (int p = tid; p < n; p += VEC_THREADS) out[p] = __ldg(src + p);
        } else {
            for (int p = tid; p < n; p += VEC_THREADS) {
                const float a = __ldg(x0 + p);
                out[p] = __fadd_rn(a, __fmul_rn(c, __fsub_rn(__ldg(xk + p), a)));
            }
        }
    }
    if (job.weights_out && tid < nin) job.weights_out[tid] = cf[tid];
}

// Randomized bucketing (rcmarl_bucket_mix, include/rcmarl.h): one CTA of VEC_THREADS threads per job.  Thread 0 draws
// the permutation into shared memory and keeps each bucket as a bit mask over the slots; the rows take one thread per
// coordinate and add each bucket's members in slot order straight from global memory (every received row is read
// once).  A bucket with a non-finite mean coordinate is found by a block-wide vote, and its row is rewritten as +inf.
struct BucketParams { rcmarl_bucket_job jobs[RCMARL_MAX_JOBS]; };

// The received messages of a bucketing job, read from global memory: message k at msgs + in_nodes[k] * stride.
struct GlobalRows {
    const float* msgs;
    const int32_t* in_nodes;
    int64_t stride;
    __device__ __forceinline__ float at(int k, int p) const { return __ldg(msgs + (int64_t)in_nodes[k] * stride + p); }
};

// The buckets of one shuffle (one thread): pi[0:m] = the received slots 1 .. m by Fisher-Yates, i = m-1 down to 1, draw
// t = word t & 3 of Philox4x32-10 at counter (ctr.x | t >> 2, ctr.y, ctr.z, ctr.w); members[b] = bit l for each slot l
// of bucket b (pi[b*s .. (b+1)*s - 1]).  pi is shared scratch of m ints.
__device__ __forceinline__ void bucket_draw(uint4 ctr, uint2 key, int m, int s, int* pi, unsigned* members) {
    const int nb = m == 0 ? 0 : (m - 1) / s + 1;   // ceil(m / s) without overflow at a huge s
    for (int q = 0; q < m; ++q) pi[q] = q + 1;
    uint4 r = make_uint4(0u, 0u, 0u, 0u);
    for (int i = m - 1, t = 0; i >= 1; --i, ++t) {
        if ((t & 3) == 0) r = philox4x32_10(make_uint4(ctr.x | (uint32_t)(t >> 2), ctr.y, ctr.z, ctr.w), key);
        const uint32_t u = (t & 3) == 0 ? r.x : (t & 3) == 1 ? r.y : (t & 3) == 2 ? r.z : r.w;
        const int j = (int)(((uint64_t)u * (uint64_t)(i + 1)) >> 32);
        const int a = pi[i];
        pi[i] = pi[j];
        pi[j] = a;
    }
    for (int b = 0; b < nb; ++b) members[b] = 0u;
    for (int q = 0; q < m; ++q) members[q / s] |= 1u << pi[q];
}

// The bucket means of rcmarl_bucket_mix over the slots row.at(l, p), l = 1 .. nin - 1: bucket b's mean to dst(b)[0:n],
// or +inf throughout if a coordinate of it is not finite.  Called by the whole CTA of VEC_THREADS threads; each thread
// writes its own coordinates only, and the caller synchronises before reading another's.
template <class Row, class Dst>
__device__ __forceinline__ void bucket_means(const Row& row, int n, int nin, int nb, const unsigned* members,
                                             const Dst& dst) {
    const int tid = threadIdx.x;
    for (int b = 0; b < nb; ++b) {
        const unsigned mask = members[b];
        const float cnt = (float)__popc(mask);
        float* out = dst(b);
        bool bad = false;
        for (int p = tid; p < n; p += VEC_THREADS) {
            float s = 0.f;
            for (int l = 1; l < nin; ++l)
                if ((mask >> l) & 1u) s += row.at(l, p);
            const float v = s / cnt;
            bad |= !isfinite(v);
            out[p] = v;
        }
        if (__syncthreads_or(bad))
            for (int p = tid; p < n; p += VEC_THREADS) out[p] = INFINITY;
    }
}

__global__ void __launch_bounds__(VEC_THREADS) bucket_mix_kernel(const __grid_constant__ BucketParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    static_assert(MAXN * MAXN <= VEC_THREADS, "one thread per entry of M");
    __shared__ int pi[MAXN];
    __shared__ unsigned members[MAXN];             // bucket b: bit l set for slot l in the bucket
    const rcmarl_bucket_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in, m = nin - 1;
    const int nb = m == 0 ? 0 : (m - 1) / job.s + 1;
    const int tid = threadIdx.x;
    if (tid == 0)
        bucket_draw(make_uint4(0u, job.receiver | job.net << 8 | 0x20000000u, job.round, job.epoch),
                    make_uint2((uint32_t)job.seed, (uint32_t)(job.seed >> 32)), m, job.s, pi, members);
    __syncthreads();
    const float* own = job.msgs + (int64_t)job.in_nodes[0] * job.msg_stride;
    for (int p = tid; p < n; p += VEC_THREADS) job.dst[p] = __ldg(own + p);
    bucket_means(GlobalRows{job.msgs, job.in_nodes, job.msg_stride}, n, nin, nb, members,
                 [&](int b) { return job.dst + (int64_t)(1 + b) * job.msg_stride; });
    if (job.weights_out && tid < (1 + nb) * nin) {
        const int r = tid / nin, l = tid % nin;
        float w = r == 0 && l == 0 ? 1.f : 0.f;
        if (r > 0) {
            const unsigned mask = members[r - 1];
            w = ((mask >> l) & 1u) ? 1.f / (float)__popc(mask) : 0.f;
        }
        job.weights_out[tid] = w;
    }
}

// Min-max / min-sum Byzantine messages (rcmarl_adaptive_attack, include/rcmarl.h): one CTA of 256 threads per job.  The
// honest rows are staged in shared memory, then mu and d (one thread per coordinate, mu and sigma as attack_kernel).
// Every distance and inner product is summed by ONE warp as in warp_sqdist, so its value does not depend on which warp
// takes it; gamma is solved on one thread and the output takes one thread per coordinate.
struct AdaptiveParams { rcmarl_adaptive_attack_job jobs[RCMARL_MAX_JOBS]; };
constexpr int ADA_THREADS = 256;

// sum_p x_p y_p of two shared-memory vectors of n floats, in every lane of the calling warp
__device__ __forceinline__ float warp_dot(const float* x, const float* y, int n, int lane) {
    float s = 0.f;
    for (int p = lane; p < n; p += 32) s = fmaf(x[p], y[p], s);
    return warp_sum(s);
}

// the largest root of A g^2 + 2 b g + e = c, cancellation-free; 0 when c - e <= 0
__device__ __forceinline__ float adaptive_root(float A, float b, float e, float c) {
    const float m = c - e;
    if (!(m > 0.f)) return 0.f;
    const float R = sqrtf(fmaxf(fmaf(b, b, A * m), 0.f));
    return b <= 0.f ? (-b + R) / A : m / (b + R);
}

// mu, d and gamma of rcmarl_adaptive_attack (kind, dev) over the nh honest rows xs[k * n .. k * n + n) staged in shared
// memory: writes mu[0:n] and d[0:n] and calls finish(gamma) on thread 0 (the caller synchronises before reading any of
// them).  Shared scratch: dist [MAXN * MAXN] (D_kl, k != l), ek, bk [MAXN], scal [2] (a; UV: ||mu||).  Called by the
// whole CTA of ADA_THREADS threads after the rows are staged.
template <class Finish>
__device__ __forceinline__ void adaptive_gamma(const float* xs, int nh, int n, const int& kind, const int& dev, float* mu,
                                               float* d, float* dist, float* ek, float* bk, float* scal,
                                               const Finish& finish) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    constexpr int NW = ADA_THREADS / 32;
    for (int p = tid; p < n; p += ADA_THREADS) {
        float s = 0.f;
        for (int k = 0; k < nh; ++k) s += xs[k * n + p];
        const float m = s / (float)nh;
        mu[p] = m;
        if (dev == RCMARL_DEV_STD) {
            float q = 0.f;
            for (int k = 0; k < nh; ++k) q = fmaf(xs[k * n + p] - m, xs[k * n + p] - m, q);
            d[p] = -sqrtf(q / (float)nh);
        } else if (dev == RCMARL_DEV_SGN) {
            d[p] = m > 0.f ? -1.f : (m < 0.f ? 1.f : 0.f);
        }
    }
    __syncthreads();
    if (dev == RCMARL_DEV_UV) {
        if (warp == 0) {
            const float q = warp_dot(mu, mu, n, lane);
            if (lane == 0) scal[1] = isfinite(q) ? sqrtf(q) : INFINITY;
        }
        __syncthreads();
        const float nrm = scal[1];
        const bool zero = nrm == 0.f || !isfinite(nrm);
        for (int p = tid; p < n; p += ADA_THREADS) d[p] = zero ? 0.f : -mu[p] / nrm;
        __syncthreads();
    }
    // warp tasks: the unordered pairs k < l, then e_k and b_k for each k, then a
    const int n_pairs = nh * (nh - 1) / 2;
    for (int t = warp; t < n_pairs + nh + 1; t += NW) {
        if (t < n_pairs) {
            int k = 0, r = t;
            while (r >= nh - 1 - k) { r -= nh - 1 - k; ++k; }
            const int l = k + 1 + r;
            const float v = warp_sqdist(xs + k * n, xs + l * n, n, lane);
            if (lane == 0) { dist[k * MAXN + l] = v; dist[l * MAXN + k] = v; }
        } else if (t < n_pairs + nh) {
            const int k = t - n_pairs;
            const float* v = xs + k * n;
            const float e = warp_sqdist(mu, v, n, lane);
            float s = 0.f;
            for (int p = lane; p < n; p += 32) s = fmaf(mu[p] - v[p], d[p], s);
            s = warp_sum(s);
            if (lane == 0) { ek[k] = e; bk[k] = s; }
        } else {
            const float q = warp_dot(d, d, n, lane);
            if (lane == 0) scal[0] = isfinite(q) ? q : INFINITY;
        }
    }
    __syncthreads();
    if (tid == 0) {
        const float a = scal[0];
        bool ok = a > 0.f && isfinite(a);
        for (int k = 0; k < nh; ++k) ok = ok && isfinite(ek[k]) && isfinite(bk[k]);
        float g = 0.f;
        if (kind == RCMARL_ADAPT_MINMAX) {
            float c = 0.f;
            for (int k = 0; k < nh; ++k)
                for (int l = k + 1; l < nh; ++l) c = fmaxf(c, dist[k * MAXN + l]);
            if (ok && isfinite(c)) {
                g = INFINITY;
                for (int k = 0; k < nh; ++k) g = fminf(g, adaptive_root(a, bk[k], ek[k], c));
                g = fmaxf(0.f, g);
            }
        } else {
            float c = 0.f, sb = 0.f, se = 0.f;
            for (int k = 0; k < nh; ++k) {
                float s = 0.f;
                for (int l = 0; l < nh; ++l)
                    if (l != k) s += dist[k * MAXN + l];
                c = fmaxf(c, s);
                sb += bk[k];
                se += ek[k];
            }
            if (ok && isfinite(c)) g = adaptive_root((float)nh * a, sb, se, c);
        }
        if (!isfinite(g)) g = 0.f;
        finish(g);
    }
}

__global__ void __launch_bounds__(ADA_THREADS) adaptive_attack_kernel(const __grid_constant__ AdaptiveParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    extern __shared__ __align__(16) float smem[];
    __shared__ float dist[MAXN * MAXN];    // D_kl, k != l
    __shared__ float ek[MAXN], bk[MAXN];
    __shared__ float scal[2];              // a; UV: ||mu||^2, then gamma
    const rcmarl_adaptive_attack_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nh = job.n_honest;
    const int tid = threadIdx.x;
    float* xs = smem;                              // [n_honest][n]
    float* mu = smem + (int64_t)nh * n;            // [n]
    float* d = mu + n;                             // [n]
    for (int k = 0; k < nh; ++k) {
        const float* src = job.msgs + (int64_t)job.honest[k] * job.msg_stride;
        for (int p = tid; p < n; p += ADA_THREADS) xs[k * n + p] = __ldg(src + p);
    }
    __syncthreads();
    adaptive_gamma(xs, nh, n, job.kind, job.dev, mu, d, dist, ek, bk, scal, [&](float g) {
        scal[1] = g;
        if (job.gamma_out) *job.gamma_out = g;
    });
    __syncthreads();
    const float t = job.scale * scal[1];
    for (int p = tid; p < n; p += ADA_THREADS) job.dst[p] = t == 0.f ? mu[p] : fmaf(t, d[p], mu[p]);
}

// Rule-aware Byzantine messages (rcmarl_tailored_attack, include/rcmarl.h): one CTA of 256 threads per job.  The real
// slots are staged in shared memory, the honest ones first (in slot order, so that adaptive_gamma sees exactly the rows
// rcmarl_adaptive_attack would), then mu, d, the candidate row and one work row.  Every crafted slot maps to the
// candidate row, so the receiver's rule (resilient_mean_small per coordinate, or vector_rule) runs unchanged on the slot
// list x(gamma_i), once per candidate; its output goes to the work row and one warp sums the objective.
struct TailoredParams { rcmarl_tailored_attack_job jobs[RCMARL_MAX_JOBS]; };
static_assert(ADA_THREADS == VEC_THREADS, "one CTA runs both the adaptive and the vector rule bodies");

// The slot list of a tailored job: slot k at xs + off[k].
struct SlotRows {
    const float* xs;
    const int* off;
    __device__ __forceinline__ const float* operator()(int k) const { return xs + off[k]; }
    __device__ __forceinline__ float at(int k, int p) const { return xs[off[k] + p]; }
};

// Shared scratch of the tailored and pipeline searches (see adaptive_gamma and vector_rule for dist .. total).
struct TailoredShared {
    float dist[RCMARL_MAX_NEIGHBOURS * RCMARL_MAX_NEIGHBOURS];
    float ek[RCMARL_MAX_NEIGHBOURS], bk[RCMARL_MAX_NEIGHBOURS], wt[RCMARL_MAX_NEIGHBOURS], score[RCMARL_MAX_NEIGHBOURS];
    float scal[2], total, best_o;
    int off[RCMARL_MAX_NEIGHBOURS], best_i;         // slot k at xs + off[k]; the search's best objective and index
};

// The coordinate-wise rule over nrows rows: z[p] = resilient_mean_small of row(0 .. nrows - 1) at p, own = row 0.
template <class Row>
__device__ __forceinline__ void coord_rule(const Row& row, int n, int nrows, int H, int rule, float* z) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    for (int p = threadIdx.x; p < n; p += ADA_THREADS) {
        float v[MAXN];
#pragma unroll
        for (int k = 0; k < MAXN; ++k) v[k] = k < nrows ? row.at(k, p) : 0.f;
        z[p] = resilient_mean_small<MAXN>(v, nrows, H, rule);
    }
}

// Stage a tailored job's real slots at xs (the honest ones first) and point every crafted slot at cand (S.off).  Called
// by the whole CTA; the caller synchronises before reading the rows.
__device__ __forceinline__ void tailored_stage(const rcmarl_tailored_attack_job& job, int nh, float* xs, const float* cand,
                                               TailoredShared& S) {
    const int n = job.n, nin = job.n_in, tid = threadIdx.x;
    if (tid == 0) {
        int h = 0, o = nh;
        for (int k = 0; k < nin; ++k)
            S.off[k] = job.slots[k] < 0 ? (int)(cand - xs) : ((job.honest_mask >> k) & 1u ? h++ : o++) * n;
        S.best_o = -INFINITY;
        S.best_i = 0;
    }
    __syncthreads();
    for (int k = 0; k < nin; ++k) {
        if (job.slots[k] < 0) continue;
        const float* src = job.msgs + (int64_t)job.slots[k] * job.msg_stride;
        float* row = xs + S.off[k];
        for (int p = tid; p < n; p += ADA_THREADS) row[p] = __ldg(src + p);
    }
}

// mu, d and Gamma = scale * gamma_mm over the nh honest rows at xs, 0 if that fp32 product is not finite (a huge scale:
// dst = mu).  Called by the whole CTA once the rows are staged; returns Gamma in every thread.
__device__ __forceinline__ float tailored_range(const rcmarl_tailored_attack_job& job, int nh, const float* xs, float* mu,
                                                float* d, TailoredShared& S) {
    const int n = job.n;
    constexpr int kind = RCMARL_ADAPT_MINMAX;
    adaptive_gamma(xs, nh, n, kind, job.dev, mu, d, S.dist, S.ek, S.bk, S.scal, [&](float g) { S.scal[1] = g; });
    __syncthreads();
    const float prod = job.scale * S.scal[1];
    return isfinite(prod) ? prod : 0.f;
}

// tailored_stage, then tailored_range over the raw messages.  Called by the whole CTA; returns Gamma in every thread.
__device__ __forceinline__ float tailored_setup(const rcmarl_tailored_attack_job& job, int nh, float* xs, float* mu,
                                                float* d, const float* cand, TailoredShared& S) {
    tailored_stage(job, nh, xs, cand, S);
    __syncthreads();
    return tailored_range(job, nh, xs, mu, d, S);
}

// The candidate search: for i = 0 .. K, cand = m(gamma_i), then for each sample q < nq eval(q) writes the modelled
// aggregate R_q(gamma_i) to z[0:n] and warp 0 sums O_i,q; Obar_i = (sum_q O_i,q in q order, from 0) / nq, -inf once an
// O_i,q or Obar_i is not finite (at nq = 1, Obar_i = O_i bitwise).  Called by the whole CTA after tailored_setup;
// returns i* (ties to the smaller i) in every thread.
template <class Eval>
__device__ __forceinline__ int tailored_search(const float* mu, const float* d, float* cand, const float* z, int n,
                                               float range, int nq, TailoredShared& S, const Eval& eval) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = 0; i <= RCMARL_TAILORED_STEPS; ++i) {
        const float g = range * (float)i / (float)RCMARL_TAILORED_STEPS;
        for (int p = tid; p < n; p += ADA_THREADS) cand[p] = g == 0.f ? mu[p] : fmaf(g, d[p], mu[p]);
        float acc = 0.f;                                              // warp 0: sum_q O_i,q
        for (int q = 0; q < nq; ++q) {
            __syncthreads();                                          // x(gamma_i) complete; the last objective read
            eval(q);
            __syncthreads();                                          // R_q(x(gamma_i)) complete
            if (warp == 0) {                                          // O_i,q = sum_p (R_p - mu_p)^2, one warp
                float s = 0.f;
                for (int p = lane; p < n; p += 32) {
                    const float e = z[p] - mu[p];
                    s = fmaf(e, e, s);
                }
                s = warp_sum(s);
                acc = isfinite(s) ? acc + s : -INFINITY;              // not finite: -inf, and -inf stays
            }
        }
        const float o = acc / (float)nq;
        if (tid == 0 && isfinite(o) && o > S.best_o) {                // ties to the smaller i
            S.best_o = o;
            S.best_i = i;
        }
    }
    __syncthreads();
    return S.best_i;
}

// (at most one CTA per job and 117 KB of staging per CTA: the register budget of one CTA per SM keeps it free of spills)
__global__ void __launch_bounds__(ADA_THREADS, 1) tailored_attack_kernel(const __grid_constant__ TailoredParams P) {
    extern __shared__ __align__(16) float smem[];
    __shared__ TailoredShared S;
    const rcmarl_tailored_attack_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    int nh = 0, nr = 0;                            // honest slots, real slots
    for (int k = 0; k < nin; ++k) {
        nh += (job.honest_mask >> k) & 1u;
        nr += job.slots[k] >= 0 ? 1 : 0;
    }
    float* xs = smem;                              // [nr][n]: the honest slots, then the other real slots
    float* mu = smem + (int64_t)nr * n;            // [n]
    float* d = mu + n;                             // [n]
    float* cand = d + n;                           // [n]: m(gamma_i), every crafted slot
    float* z = cand + n;                           // [n]: the rule's output (and GMED's iterate)
    const float range = tailored_setup(job, nh, xs, mu, d, cand, S);
    const SlotRows rows{xs, S.off};
    const int best = tailored_search(mu, d, cand, z, n, range, 1, S, [&](int) {
        if (job.family == RCMARL_TAILOR_COORD)
            coord_rule(rows, n, nin, job.H, job.rule, z);
        else
            vector_rule(rows, n, nin, job.H, job.rule, z, z, S.dist, S.wt, S.score, S.total);
    });
    const float g = range * (float)best / (float)RCMARL_TAILORED_STEPS;
    if (tid == 0 && job.gamma_out) *job.gamma_out = g;
    for (int p = tid; p < n; p += ADA_THREADS) job.dst[p] = g == 0.f ? mu[p] : fmaf(g, d[p], mu[p]);
}

// Pipeline-aware Byzantine messages (rcmarl_pipeline_attack, include/rcmarl.h): tailored_attack_kernel's staging and
// search, with the receiver's mixing step before its rule.  Behind the real slots, mu, d, the candidate and the output
// row come the mixed rows (nnm: n_in; bucketing: the bucket means, the own row being read in place), and for DnC the
// fp64 mean sits in front, 8-byte aligned.  The mixing and the rule read their rows through slot offsets, so one
// instantiation of each body serves every mixing.  The attacker's bucketing shuffles are drawn once per job by thread 0.
struct PipelineParams { rcmarl_pipeline_attack_job jobs[RCMARL_MAX_JOBS]; };
static_assert(ADA_THREADS == VEC_THREADS, "dnc_rule, nnm_rows, bucket_means and vector_rule stride by VEC_THREADS");

// The receiver's ARC step inside the ARC forms of the pipeline and history searches (rcmarl_pipeline_arc_attack,
// rcmarl_history_arc_attack): d_k and c_k of each slot, and the row the next stage reads for slot k at xs + off[k].
struct ArcShared {
    float dist[RCMARL_MAX_NEIGHBOURS], cf[RCMARL_MAX_NEIGHBOURS], tau;
    int off[RCMARL_MAX_NEIGHBOURS];
};

// dist[k] = d_k = sqrtf(squared distance of slot k's row and slot 0's) for each slot k >= 1 of `mask`, each summed by
// ONE warp with warp_sqdist as in arc_clip_kernel (slot k's row at xs + off[k]).  Called by the whole CTA; the caller
// synchronises before reading dist.
__device__ __forceinline__ void arc_dist(const float* xs, const int* off, int n, int nin, unsigned mask, float* dist) {
    constexpr int NW = ADA_THREADS / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int k = 1 + warp; k < nin; k += NW)
        if ((mask >> k) & 1u) {
            const float d = sqrtf(warp_sqdist(xs + off[k], xs + off[0], n, lane));
            if (lane == 0) dist[k] = d;
        }
}

// ARC of one candidate, called by the whole CTA once the slot rows (slot k at xs + off[k], slot 0 real) are complete and
// A.dist holds d_k of every slot whose row does not depend on the candidate: d_k of the slots of `sum` is summed here,
// each slot of `copy` takes d_from's; then the factors (arc_factors) and A.off[k]: slot k's own row if c_k = 1, slot 0's
// if c_k = 0, else a row of its own in clip (at most k_clip of them), x_0 + c_k (x_k - x_0) with every operation rounded
// on its own (arc_clip_kernel's arithmetic).  The clipped rows are complete on return.
__device__ __forceinline__ void arc_rows(float* xs, const int* off, int n, int nin, int H, unsigned sum, unsigned copy,
                                         int from, float* clip, ArcShared& A) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    arc_dist(xs, off, n, nin, sum, A.dist);
    __syncthreads();
    if (warp == 0) {
        if (lane < nin && ((copy >> lane) & 1u)) A.dist[lane] = A.dist[from];
        __syncwarp();
        arc_factors(A.dist, nin, H, A.tau, A.cf, lane);
        __syncwarp();
        if (lane == 0)
            for (int k = 0, c = 0; k < nin; ++k) {
                const float ck = A.cf[k];
                A.off[k] = ck == 1.f ? off[k] : ck == 0.f ? off[0] : (int)(clip - xs) + n * c++;
            }
    }
    __syncthreads();
    const float* x0 = xs + off[0];
    for (int k = 1; k < nin; ++k) {
        const float c = A.cf[k];
        if (c == 1.f || c == 0.f) continue;
        const float* xk = xs + off[k];
        float* out = xs + A.off[k];
        for (int p = tid; p < n; p += ADA_THREADS) {
            const float a = x0[p];
            out[p] = __fadd_rn(a, __fmul_rn(c, __fsub_rn(xk[p], a)));
        }
    }
    __syncthreads();
}

// The receiver's MDA / SMEA rule inside the subset forms of the pipeline and history searches
// (rcmarl_subset_pipeline_attack, rcmarl_subset_history_attack): subset_rule's scratch, and the flags and pairwise
// distances of the rows that do not depend on the candidate (subset_known), taken once per job.
struct SubsetAttackShared {
    SubsetShared S;
    double DK[RCMARL_MAX_NEIGHBOURS * RCMARL_MAX_NEIGHBOURS];
    int flag[RCMARL_MAX_NEIGHBOURS];
    SubsetKnownBest KB;
};

// The receiver's rule stage in the pipeline and history searches: the base rules (families COORD, VECTOR and
// SPECTRAL), MDA / SMEA (the subset forms, subset_rule) or IOS (the IOS forms, ios_rule, whose fp64 centre takes the
// region in front of the real slots that DnC's mean takes).
enum RuleStage { STAGE_BASE = 0, STAGE_SUBSET = 1, STAGE_IOS = 2 };

template <bool ARC, int STAGE>
__global__ void __launch_bounds__(ADA_THREADS, 1) pipeline_attack_kernel(const __grid_constant__ PipelineParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr bool SUBSET = STAGE == STAGE_SUBSET, IOS = STAGE == STAGE_IOS;
    extern __shared__ __align__(16) float smem[];
    __shared__ TailoredShared S;
    __shared__ DncShared D;
    __shared__ unsigned sel[MAXN];                                   // nnm: N_k
    __shared__ unsigned members[RCMARL_PIPELINE_MAX_PERMS * MAXN];   // bucketing: bucket b of sample q at [q * MAXN + b]
    __shared__ int pi[MAXN];
    __shared__ int roff[MAXN];                                       // the rule's row k at xs + roff[k]
    __shared__ ArcShared A;                                          // ARC
    const rcmarl_pipeline_attack_job& pj = P.jobs[blockIdx.x];
    const rcmarl_tailored_attack_job& job = pj.attack;
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    const bool bucket = pj.mixing == RCMARL_PIPE_BUCKET;
    const int nb = bucket ? (nin - 2) / pj.s + 1 : 0;                // ceil((n_in - 1) / s); n_in >= 2
    const int nrows = bucket ? 1 + nb : nin, nq = bucket ? pj.n_perms : 1;
    int nh = 0, nr = 0;                            // honest slots, real slots
    for (int k = 0; k < nin; ++k) {
        nh += (job.honest_mask >> k) & 1u;
        nr += job.slots[k] >= 0 ? 1 : 0;
    }
    double* mu64 = reinterpret_cast<double*>(smem);                 // DnC, IOS: [n]
    float* xs = smem + (IOS || job.family == RCMARL_TAILOR_SPECTRAL ? 2 * (int64_t)n : 0);   // [nr][n]
    float* mu = xs + (int64_t)nr * n;              // [n]
    float* d = mu + n;                             // [n]
    float* cand = d + n;                           // [n]: m(gamma_i), every crafted slot
    float* z = cand + n;                           // [n]: the rule's output (and GMED's iterate)
    float* mixed = z + n;                          // nnm: [n_in][n]; bucketing: [nb][n]; then ARC: [k_clip][n]
    const int n_mixed = pj.mixing == RCMARL_PIPE_NNM ? nin : nb;
    if (tid == 0 && bucket)
        for (int q = 0; q < nq; ++q)
            bucket_draw(make_uint4((uint32_t)q << 2, pj.attacker | pj.receiver << 8 | pj.net << 16 | 0x10000000u,
                                   pj.round, pj.epoch),
                        make_uint2((uint32_t)pj.seed, (uint32_t)(pj.seed >> 32)), nin - 1, pj.s, pi, members + q * MAXN);
    const float range = tailored_setup(job, nh, xs, mu, d, cand, S);
    if (tid == 0) {
        const int base = (int)(mixed - xs);
        for (int k = 0; k < nrows; ++k)
            roff[k] = pj.mixing == RCMARL_PIPE_NONE ? S.off[k] : pj.mixing == RCMARL_PIPE_NNM ? base + k * n
                    : k == 0 ? S.off[0] : base + (k - 1) * n;
    }
    __syncthreads();
    const int *soff = S.off, *ooff = roff;        // the rows the mixing step and the rule read
    unsigned real = 0u;                           // ARC: the real slots, and the first crafted one
    int from = 0;
    if constexpr (ARC) {
        for (int k = nin - 1; k >= 0; --k)
            if (job.slots[k] >= 0) real |= 1u << k;
            else from = k;
        arc_dist(xs, S.off, n, nin, real, A.dist);  // the real slots' d_k, once per job
        soff = A.off;
        if (pj.mixing == RCMARL_PIPE_NONE) ooff = A.off;
    }
    const SlotRows slots{xs, soff}, rows{xs, ooff};
    SubsetAttackShared* U = nullptr;              // SUBSET: the rule's scratch
    unsigned known = 0u;                          // SUBSET: the rule's rows that do not depend on the candidate
    if constexpr (SUBSET) {
        __shared__ SubsetAttackShared SU;
        U = &SU;
        subset_binom(SU.S);
        if (!ARC && pj.mixing == RCMARL_PIPE_NONE) {   // the real slots: their flags and distances once per job
            for (int k = 0; k < nin; ++k) known |= job.slots[k] >= 0 ? 1u << k : 0u;
            subset_known(rows, n, nin, known, SU.flag, SU.DK);
        }
        if (tid == 0) SU.KB.urows = 0u;
        __syncthreads();
    }
    IosShared* I = nullptr;                       // IOS: the rule's scratch
    if constexpr (IOS) {
        __shared__ IosShared IS;
        I = &IS;
    }
    const auto eval = [&](int q) {
        if constexpr (ARC)                        // once per candidate: every crafted slot holds it, one d_k for all
            if (q == 0)
                arc_rows(xs, S.off, n, nin, job.H, 1u << from, ~real & ~(1u << from) & ((1u << nin) - 1u), from,
                         mixed + (int64_t)n_mixed * n, A);
        if (pj.mixing == RCMARL_PIPE_NNM) {
            nnm_rows(slots, n, nin, job.H, S.dist, sel, [&](int k) { return mixed + k * n; });
            __syncthreads();                                          // the mixed rows complete
        } else if (bucket) {
            bucket_means(slots, n, nin, nb, members + q * MAXN, [&](int b) { return mixed + b * n; });
            __syncthreads();
        }
        if constexpr (SUBSET)
            subset_rule(rows, n, nrows, job.H, job.rule, z, U->S, known, U->flag, U->DK, known ? &U->KB : nullptr);
        else if constexpr (IOS)
            ios_rule(rows, n, nrows, job.H, mu64, z, *I);
        else if (job.family == RCMARL_TAILOR_COORD)
            coord_rule(rows, n, nrows, job.H, job.rule, z);
        else if (job.family == RCMARL_TAILOR_VECTOR)
            vector_rule(rows, n, nrows, job.H, job.rule, z, z, S.dist, S.wt, S.score, S.total);
        else
            dnc_rule(rows, n, nrows, job.H, mu64, z, D);
    };
    const int best = tailored_search(mu, d, cand, z, n, range, nq, S, eval);
    const float g = range * (float)best / (float)RCMARL_TAILORED_STEPS;
    if (tid == 0 && job.gamma_out) *job.gamma_out = g;
    for (int p = tid; p < n; p += ADA_THREADS) {
        const float v = g == 0.f ? mu[p] : fmaf(g, d[p], mu[p]);
        job.dst[p] = v;
        cand[p] = v;
    }
    if (pj.model_out) {                            // R_0(gamma_i*), the same for every thread of the CTA
        __syncthreads();
        eval(0);
        __syncthreads();
        for (int p = tid; p < n; p += ADA_THREADS) pj.model_out[p] = z[p];
    }
}

// Dissensus messages (rcmarl_dissensus_attack, include/rcmarl.h): one thread per coordinate, as attack_kernel; the
// honest pull delta is summed in list order from 0.
struct DissensusParams { rcmarl_dissensus_job jobs[RCMARL_MAX_JOBS]; };
__global__ void __launch_bounds__(256) dissensus_attack_kernel(const __grid_constant__ DissensusParams P) {
    const rcmarl_dissensus_job& job = P.jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= job.n) return;
    const float x = __ldg(job.msgs + (int64_t)job.own * job.msg_stride + i);
    float delta = 0.f;
    for (int k = 0; k < job.n_honest; ++k) delta += __ldg(job.msgs + (int64_t)job.honest[k] * job.msg_stride + i) - x;
    const float c = job.eps / (float)job.n_byz;
    job.dst[i] = c == 0.f ? x : fmaf(-c, delta, x);
}

// Per-neighbour momentum (rcmarl_momentum_mix, include/rcmarl.h): one thread per coordinate, blockIdx.z the slot.  Every
// operation is rounded on its own (__f*_rn), so no FMA is contracted and an fp32 NumPy restatement matches bitwise.
struct MomentumParams { rcmarl_momentum_job jobs[RCMARL_MAX_JOBS]; };

// One coordinate of one slot's momentum step: M' at u = x - c, the old M at *m (read only when !first).  Shared by
// momentum_mix_kernel and history_attack_kernel, so that the attacker's model is the receiver's arithmetic.
__device__ __forceinline__ float momentum_next(float u, const float* m, float beta, int first) {
    float v = u;
    if (!first) {
        const float old = *m;
        if (isinf(old)) v = old;
        else if (isfinite(u)) v = __fadd_rn(__fmul_rn(beta, old), __fmul_rn(__fsub_rn(1.f, beta), u));
    }
    return v;
}

__global__ void __launch_bounds__(256) momentum_mix_kernel(const __grid_constant__ MomentumParams P) {
    const rcmarl_momentum_job& job = P.jobs[blockIdx.y];
    const int k = blockIdx.z;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= job.n_in || i >= job.n) return;
    const float c = __ldg(job.ref + i);
    const float u = __fsub_rn(__ldg(job.msgs + (int64_t)job.in_nodes[k] * job.msg_stride + i), c);
    float* m = job.momentum + (int64_t)k * job.momentum_stride + i;
    const float v = momentum_next(u, m, job.beta, job.first);
    *m = v;
    job.dst[(int64_t)k * job.msg_stride + i] = __fadd_rn(c, v);
}

// Momentum-aware Byzantine messages (rcmarl_history_attack, include/rcmarl.h): pipeline_attack_kernel without mixing,
// in momentum-row space.  The real slots are staged by tailored_stage and stepped in place before mu, d and gamma_mm
// are taken; behind mu, d, the target and the output row come one row per crafted slot (colluders' rows differ), and
// for DnC the fp64 mean sits in front, 8-byte aligned.  A crafted slot's M row is read from global memory for each
// candidate.
struct HistoryParams { rcmarl_history_attack_job jobs[RCMARL_MAX_JOBS]; };

// the message that puts a slot's momentum row at t (include/rcmarl.h, Inversion); m is read only when !first
__device__ __forceinline__ float momentum_invert(float t, float c, const float* m, float beta, int first) {
    if (first) return t;
    const float old = *m;
    if (isinf(old)) return t;
    return __fadd_rn(c, __fdiv_rn(__fsub_rn(__fsub_rn(t, c), __fmul_rn(beta, old)), __fsub_rn(1.f, beta)));
}

template <bool ARC, int STAGE>
__global__ void __launch_bounds__(ADA_THREADS, 1) history_attack_kernel(const __grid_constant__ HistoryParams P) {
    constexpr bool SUBSET = STAGE == STAGE_SUBSET, IOS = STAGE == STAGE_IOS;
    extern __shared__ __align__(16) float smem[];
    __shared__ TailoredShared S;
    __shared__ DncShared D;
    __shared__ ArcShared A;                        // ARC
    const rcmarl_history_attack_job& hj = P.jobs[blockIdx.x];
    const rcmarl_tailored_attack_job& job = hj.attack;
    const int n = job.n, nin = job.n_in;
    const int tid = threadIdx.x;
    int nh = 0, nr = 0;                            // honest slots, real slots
    for (int k = 0; k < nin; ++k) {
        nh += (job.honest_mask >> k) & 1u;
        nr += job.slots[k] >= 0 ? 1 : 0;
    }
    const int k0 = __ffs(hj.own_mask) - 1;         // the lowest own slot
    double* mu64 = reinterpret_cast<double*>(smem);                 // DnC, IOS: [n]
    float* xs = smem + (IOS || job.family == RCMARL_TAILOR_SPECTRAL ? 2 * (int64_t)n : 0);   // [nr][n]
    float* mu = xs + (int64_t)nr * n;              // [n]
    float* d = mu + n;                             // [n]
    float* cand = d + n;                           // [n]: the target t(gamma_i)
    float* z = cand + n;                           // [n]: the rule's output (and GMED's iterate)
    float* crafted = z + n;                        // [n_in - nr][n]: a_k of each crafted slot, in slot order
    float* clip = crafted + (int64_t)(nin - nr) * n;   // ARC: [k_clip][n]
    tailored_stage(job, nh, xs, cand, S);
    if (tid == 0)                                  // each crafted slot to a row of its own
        for (int k = 0, c = 0; k < nin; ++k)
            if (job.slots[k] < 0) S.off[k] = (int)(crafted - xs) + n * c++;
    __syncthreads();
    const auto Mrow = [&](int k) { return hj.momentum + (int64_t)k * hj.momentum_stride; };
    for (int k = 0; k < nin; ++k) {                // r_k = step_k(x_k) in place
        if (job.slots[k] < 0) continue;
        float* row = xs + S.off[k];
        const float* m = Mrow(k);
        for (int p = tid; p < n; p += ADA_THREADS) {
            const float c = __ldg(hj.ref + p);
            row[p] = __fadd_rn(c, momentum_next(__fsub_rn(row[p], c), m + p, hj.beta, hj.first));
        }
    }
    __syncthreads();
    unsigned real = 0u;                            // ARC: the real slots
    if constexpr (ARC) {
        for (int k = 0; k < nin; ++k) real |= job.slots[k] >= 0 ? 1u << k : 0u;
        arc_dist(xs, S.off, n, nin, real, A.dist); // the real slots' d_k, once per job
    }
    const float range = tailored_range(job, nh, xs, mu, d, S);
    const SlotRows rows{xs, ARC ? A.off : S.off};
    SubsetAttackShared* U = nullptr;               // SUBSET: the rule's scratch
    unsigned known = 0u;                           // SUBSET: the rule's rows that do not depend on the candidate
    if constexpr (SUBSET) {
        __shared__ SubsetAttackShared SU;
        U = &SU;
        subset_binom(SU.S);
        if (!ARC) {                                // the real slots' rows r_k: their flags and distances once per job
            for (int k = 0; k < nin; ++k) known |= job.slots[k] >= 0 ? 1u << k : 0u;
            subset_known(rows, n, nin, known, SU.flag, SU.DK);
        }
        if (tid == 0) SU.KB.urows = 0u;
        __syncthreads();
    }
    IosShared* I = nullptr;                        // IOS: the rule's scratch
    if constexpr (IOS) {
        __shared__ IosShared IS;
        I = &IS;
    }
    // a_k of every crafted slot for the target in cand, then the rule into z; returns whether every crafted message is
    // finite (the same in every thread).  An infeasible candidate skips the rule unless `always`: its objective is -inf
    // whatever the rule gives.
    const auto model = [&](bool always) {
        bool bad = false;
        for (int k = 0; k < nin; ++k) {
            if (job.slots[k] < 0) {
                float* row = xs + S.off[k];
                const float* m = Mrow(k);
                const float* src = Mrow((hj.own_mask >> k) & 1u ? k0 : k);
                for (int p = tid; p < n; p += ADA_THREADS) {
                    const float c = __ldg(hj.ref + p);
                    const float x = momentum_invert(cand[p], c, src + p, hj.beta, hj.first);
                    bad = bad || !isfinite(x);
                    row[p] = __fadd_rn(c, momentum_next(__fsub_rn(x, c), m + p, hj.beta, hj.first));
                }
            }
        }
        const bool ok = !__syncthreads_or(bad);    // the crafted rows complete
        if (!ok && !always) return false;
        if constexpr (ARC)                         // one d_k per crafted slot: colluders' rows differ
            arc_rows(xs, S.off, n, nin, job.H, ~real & ((1u << nin) - 1u), 0u, 0, clip, A);
        if constexpr (SUBSET)
            subset_rule(rows, n, nin, job.H, job.rule, z, U->S, known, U->flag, U->DK, known ? &U->KB : nullptr);
        else if constexpr (IOS)
            ios_rule(rows, n, nin, job.H, mu64, z, *I);
        else if (job.family == RCMARL_TAILOR_COORD)
            coord_rule(rows, n, nin, job.H, job.rule, z);
        else if (job.family == RCMARL_TAILOR_VECTOR)
            vector_rule(rows, n, nin, job.H, job.rule, z, z, S.dist, S.wt, S.score, S.total);
        else
            dnc_rule(rows, n, nin, job.H, mu64, z, D);
        return ok;
    };
    const int best = tailored_search(mu, d, cand, z, n, range, 1, S, [&](int) {
        // infeasible: a non-finite objective, O_i = -inf (z is not read before tailored_search's next barrier)
        if (!model(false) && tid == 0) z[0] = INFINITY;
    });
    const float g = range * (float)best / (float)RCMARL_TAILORED_STEPS;
    if (tid == 0 && job.gamma_out) *job.gamma_out = g;
    const float* m0 = Mrow(k0);
    for (int p = tid; p < n; p += ADA_THREADS) {
        const float t = g == 0.f ? mu[p] : fmaf(g, d[p], mu[p]);
        job.dst[p] = momentum_invert(t, __ldg(hj.ref + p), m0 + p, hj.beta, hj.first);
        cand[p] = t;
    }
    if (hj.model_out) {                            // R(gamma_i*), the same for every thread of the CTA
        __syncthreads();
        model(true);
        __syncthreads();
        for (int p = tid; p < n; p += ADA_THREADS) hj.model_out[p] = z[p];
    }
}

// Mimic messages (rcmarl_mimic_attack, include/rcmarl.h): one CTA of 256 threads per job.  The honest rows are staged
// in shared memory and centred in place (mu as attack_kernel), next to mu, z and u.  Every sum over p is taken by ONE
// warp (warp_dot), so its value does not depend on which warp takes it; the per-row sums are spread over the warps, the
// choices run on thread 0 and the elementwise steps take one thread per coordinate.
struct MimicParams { rcmarl_mimic_job jobs[RCMARL_MAX_JOBS]; };

__global__ void __launch_bounds__(ADA_THREADS) mimic_attack_kernel(const __grid_constant__ MimicParams P) {
    constexpr int MAXN = RCMARL_MAX_NEIGHBOURS;
    constexpr int NW = ADA_THREADS / 32;
    extern __shared__ __align__(16) float smem[];
    __shared__ float sk[MAXN];                     // e_k (Init), s_k (Step), t_k (Choose)
    __shared__ float scal;                         // the divisor sqrtf(e_k0) or sqrtf(q)
    __shared__ int pick, live;                     // k0 / k*; whether z is to be rescaled
    const rcmarl_mimic_job& job = P.jobs[blockIdx.x];
    const int n = job.n, nh = job.n_honest;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float* cs = smem;                              // [n_honest][n]: c_k = v_k - mu
    float* mu = smem + (int64_t)nh * n;            // [n]
    float* z = mu + n;                             // [n]
    float* u = z + n;                              // [n]
    for (int k = 0; k < nh; ++k) {
        const float* src = job.msgs + (int64_t)job.honest[k] * job.msg_stride;
        for (int p = tid; p < n; p += ADA_THREADS) cs[k * n + p] = __ldg(src + p);
    }
    int nonzero = 0;
    for (int p = tid; p < n; p += ADA_THREADS) {
        const float v = job.z[p];
        z[p] = v;
        nonzero |= v != 0.f;
    }
    __syncthreads();
    for (int p = tid; p < n; p += ADA_THREADS) {
        float s = 0.f;
        for (int k = 0; k < nh; ++k) s += cs[k * n + p];
        const float m = s / (float)nh;
        mu[p] = m;
        for (int k = 0; k < nh; ++k) cs[k * n + p] = cs[k * n + p] - m;
    }
    bool zero = !__syncthreads_or(nonzero);
    if (zero) {                                                       // Init: the largest centred row, normalised
        for (int k = warp; k < nh; k += NW) {
            const float e = warp_dot(cs + k * n, cs + k * n, n, lane);
            if (lane == 0) sk[k] = isfinite(e) ? e : INFINITY;
        }
        __syncthreads();
        if (tid == 0) {
            int k0 = 0;
            for (int k = 1; k < nh; ++k)
                if (sk[k] > sk[k0]) k0 = k;
            const float e = sk[k0];
            live = e > 0.f && isfinite(e);
            pick = k0;
            scal = sqrtf(e);
        }
        __syncthreads();
        int set = 0;
        if (live) {
            const float* c = cs + pick * n;
            const float r = scal;
            for (int p = tid; p < n; p += ADA_THREADS) {
                const float v = c[p] / r;
                z[p] = v;
                set |= v != 0.f;
            }
        }
        zero = !__syncthreads_or(set);
    }
    if (job.update == 1 && !zero) {                                  // Step: z <- C^T C z / ||C^T C z||
        for (int k = warp; k < nh; k += NW) {
            const float s = warp_dot(cs + k * n, z, n, lane);
            if (lane == 0) sk[k] = isfinite(s) ? s : INFINITY;
        }
        __syncthreads();
        for (int p = tid; p < n; p += ADA_THREADS) {
            float a = 0.f;
            for (int k = 0; k < nh; ++k) a = fmaf(sk[k], cs[k * n + p], a);
            u[p] = a;
        }
        __syncthreads();
        if (warp == 0) {
            const float q = warp_dot(u, u, n, lane);
            if (lane == 0) {
                const float qq = isfinite(q) ? q : INFINITY;
                live = qq > 0.f && isfinite(qq);
                scal = sqrtf(qq);
            }
        }
        __syncthreads();
        if (live) {
            const float r = scal;
            for (int p = tid; p < n; p += ADA_THREADS) z[p] = u[p] / r;
        }
        __syncthreads();
    }
    // Choose: the candidate furthest along z (ties to the smaller k; not finite: -inf)
    if (!zero) {
        for (int k = warp; k < nh; k += NW) {
            if (!((job.candidate_mask >> k) & 1u)) continue;
            const float t = warp_dot(cs + k * n, z, n, lane);
            if (lane == 0) sk[k] = isfinite(t) ? t : -INFINITY;
        }
    }
    __syncthreads();
    if (tid == 0) {
        int best = __ffs((int)job.candidate_mask) - 1;                // the lowest candidate
        if (!zero) {
            float bt = -INFINITY;
            for (int k = 0; k < nh; ++k)
                if (((job.candidate_mask >> k) & 1u) && sk[k] > bt) {
                    bt = sk[k];
                    best = k;
                }
        }
        pick = best;
        if (job.target_out) *job.target_out = best;
    }
    __syncthreads();
    const float* src = job.msgs + (int64_t)job.honest[pick] * job.msg_stride;
    for (int p = tid; p < n; p += ADA_THREADS) {
        job.dst[p] = __ldg(src + p);
        job.z[p] = z[p];
    }
}

struct SgdParams { rcmarl_sgd_job jobs[RCMARL_MAX_JOBS]; };
__global__ void __launch_bounds__(256) sgd_kernel(const __grid_constant__ SgdParams P) {
    const rcmarl_sgd_job& job = P.jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < job.n) {
        const float s = job.src[i];
        job.dst[i] = i >= job.first ? s - job.coef * job.sums[i - job.first] : s;
    }
    if (i == 0 && job.loss_out) {
        const float l = job.loss_coef * job.sums[job.n - job.first];
        *job.loss_out = job.loss_accumulate ? *job.loss_out + l : l;
    }
}

struct AdamParams { rcmarl_adam_job jobs[RCMARL_MAX_JOBS]; };
__global__ void __launch_bounds__(256) adam_kernel(const __grid_constant__ AdamParams P) {
    const rcmarl_adam_job& job = P.jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < job.n) {
        const float g = job.grad_scale * job.sums[i];
        const float m = job.beta1 * job.m[i] + (1.f - job.beta1) * g;
        const float v = job.beta2 * job.v[i] + (1.f - job.beta2) * g * g;
        job.m[i] = m;
        job.v[i] = v;
        job.theta[i] = job.theta[i] - job.lr_t * m / (sqrtf(v) + job.eps);
    }
    if (i == 0 && job.loss_out) {
        const float l = job.loss_coef * job.sums[job.n];
        *job.loss_out = job.loss_accumulate ? *job.loss_out + l : l;
    }
}

struct MixParams { int32_t agents[RCMARL_MAX_JOBS]; };
__global__ void __launch_bounds__(256) reward_mix_kernel(const float* __restrict__ r, int64_t n_rows, int n_agents,
                                                         const __grid_constant__ MixParams P, int n_listed,
                                                         float scale, float* __restrict__ out) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    const float inv = (float)n_listed;
    float s = 0.f;
    for (int k = 0; k < n_listed; ++k) s = s + __ldg(r + row * n_agents + P.agents[k]) / inv;  // train_agents.py:98
    out[row] = scale * s;
}

// ============================================================================================
// host-side launchers
// ============================================================================================
template <typename K>
static int set_smem(K kernel, size_t bytes) {
    if (bytes > 48 * 1024) RC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return 0;
}

static int check_rows(const rcmarl_rows* r) {
    if (!r || !r->sa || !r->ns || !r->r || r->n_rows < 0 || r->n_envs <= 0) return RCMARL_ERR_ARG;
    if (r->n_agents != 5 && r->n_agents != 16) return RCMARL_ERR_ARG;
    if (r->time_idx && (r->n_rows % r->n_envs) != 0) return RCMARL_ERR_ARG;
    return 0;
}

template <int NA>
static int launch_values(const ValuesParams& P, int n_jobs, cudaStream_t st) {
    const size_t smem = sizeof(float) * round4(param_count(3 * NA, 1) > param_count(2 * NA, NACT)
                                                   ? param_count(3 * NA, 1) : param_count(2 * NA, NACT));
    if (set_smem(values_kernel<NA>, smem)) return RCMARL_ERR_CUDA;
    int64_t gx = (P.rows.n_rows + 255) / 256;
    const int64_t cap = (int64_t)sm_count_cached() * 2;   // 2 resident CTAs per SM (126 registers x 256 threads)
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    values_kernel<NA><<<dim3((unsigned)gx, n_jobs), 256, smem, st>>>(P);
    RC_CUDA(cudaGetLastError());
    return 0;
}

// Launch as a programmatic dependent of the kernel before it on the stream, so that its grid is queued while the
// producer's last CTAs drain; the kernel waits for that grid itself (pdl_wait, griddepcontrol.wait) before it reads
// the producer's output.
template <typename K, typename Params>
static int launch_pdl(K kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Params& P) {
    cudaLaunchAttribute pdl;
    pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    pdl.val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = &pdl;
    cfg.numAttrs = 1;
    RC_CUDA(cudaLaunchKernelEx(&cfg, kernel, P));
    RC_CUDA(cudaGetLastError());
    return 0;
}

template <int NA, int LOSS>
static int launch_grad(const GradParams& P, int n_ctas, cudaStream_t st) {
    constexpr size_t smem = grad_smem_bytes<NA, LOSS>();
    static_assert(smem <= 227 * 1024, "grad kernel exceeds the 227 KB shared-memory limit");
    static bool attr = false;                          // opt-in to > 48 KB dynamic shared memory once per process
    if (!attr) {
        if (set_smem(grad_kernel<NA, LOSS>, smem)) return RCMARL_ERR_CUDA;
        attr = true;
    }
    return launch_pdl(grad_kernel<NA, LOSS>, dim3(n_ctas), dim3(32 * grad_warps<NA, LOSS>()), smem, st, P);
}

template <int NA>
static int launch_team(const TeamParams& P, int n_list, int gy, cudaStream_t st) {
    const size_t smem = sizeof(float) * (round4(param_count(3 * NA, 1)) + RCMARL_MAX_NEIGHBOURS * 24 + 8 * TEAM_N);
    if (set_smem(team_kernel<NA>, smem)) return RCMARL_ERR_CUDA;
    team_kernel<NA><<<dim3(n_list, gy), 128, smem, st>>>(P);
    RC_CUDA(cudaGetLastError());
    return 0;
}

// Sum the CTA partials of n_jobs jobs (Q.n[j] <= max_n floats each) into Q.sums: reduce_kernel, or, with a bound
// exchange context, reduce_comm_kernel, which also sums over the ranks.  Returns an RCMARL status.
static int reduce_partials(const ReduceParams& Q, int n_jobs, int max_n, cudaStream_t st) {
    if (!comm_bound()) {
        reduce_kernel<<<dim3((max_n + 31) / 32, n_jobs), 256, 0, st>>>(Q);
        RC_CUDA(cudaGetLastError());
        return RCMARL_OK;
    }
    ReduceCommParams C;
    if (!comm_next(&C.comm, (int64_t)n_jobs * max_n)) return RCMARL_ERR_ARG;
    C.partial = Q.partial; C.slots = Q.slots; C.out_stride = max_n; C.n_jobs = n_jobs; C.max_n = max_n;
    for (int j = 0; j < n_jobs; ++j) { C.sums[j] = Q.sums[j]; C.n[j] = Q.n[j]; }
    const int items = ((max_n + 31) / 32) * n_jobs, cap = sm_count_cached() * 2;    // up to two resident CTAs per SM
    return launch_pdl(reduce_comm_kernel, dim3(items < cap ? items : cap), dim3(256), 0, st, C);
}

static int grid_y_for(int64_t work_items, int n_jobs, int ctas_per_sm) {
    // one resident wave at most: gridDim.x * gridDim.y <= SMs * CTAs-per-SM (a partial second wave would
    // double the kernel time of these persistent, equal-work CTAs)
    int64_t cap = ((int64_t)sm_count_cached() * ctas_per_sm) / n_jobs;
    if (cap < 1) cap = 1;
    int64_t gy = work_items < cap ? work_items : cap;
    return (int)(gy < 1 ? 1 : gy);
}

// Shares of a one-wave grid over n jobs: g[j] = CTAs of job j; pure host arithmetic (also behind rcmarl_grad_grid_plan
// for the CPU tests).
//   balanced = false: equal shares, floor(SMs / n_jobs) CTAs per job (leaves SMs % n_jobs SMs idle, and the cheaper
//     jobs' CTAs idle at the end of the launch).
//   balanced = true (rcmarl_grad, rcmarl_minibatch_fit): shares sized by cost.  A job's cost per row depends on its
//     network (grad_row_cost) and a CTA works in rounds of `gw` 64-row chunks; greedy: the job that currently finishes
//     last gets the next CTA.  The fit kernels do ~2 000 FMA per 64-byte buffer row, so the full-batch launch reads its
//     rows at ~15 % of HBM bandwidth even with no L2 reuse between jobs; sweeping the jobs in lock-step (equal shares)
//     was measured slower than these shares (C2 fit launch 12.34 -> 12.05 ms on an H100 SXM, DESIGN.md 4.2).
static void plan_shares(int n, const int* cost, int64_t nchunks, int gw, int sms, bool balanced, int* g) {
    int64_t units = (nchunks + gw - 1) / gw;
    if (units < 1) units = 1;
    if (!balanced || n == 1 || n > sms) {
        int64_t gy = sms / n;
        if (gy < 1) gy = 1;
        if (gy > units) gy = units;
        for (int j = 0; j < n; ++j) g[j] = (int)gy;
    } else {
        int used = n;
        for (int j = 0; j < n; ++j) g[j] = 1;
        while (used < sms) {
            int best = -1;
            int64_t best_t = -1;
            for (int j = 0; j < n; ++j) {
                if (g[j] >= units) continue;
                const int64_t per_round = (int64_t)g[j] * gw;
                const int64_t t = ((nchunks + per_round - 1) / per_round) * cost[j];
                if (t > best_t || (t == best_t && g[j] < g[best])) { best_t = t; best = j; }
            }
            if (best < 0) break;
            ++g[best];
            ++used;
        }
    }
}

// 1-D grid of grad_kernel / mb_persist_kernel with the plan_shares shares: job j owns the CTAs
// [cta_first[j], cta_first[j + 1]).  Returns the CTA count.
static int plan_grid(int n, const int* cost, int64_t nchunks, int gw, bool balanced, int16_t* cta_first) {
    int g[RCMARL_MAX_JOBS];
    plan_shares(n, cost, nchunks, gw, sm_count_cached(), balanced, g);
    int first = 0;
    for (int j = 0; j < n; ++j) {
        cta_first[j] = (int16_t)first;
        first += g[j];
    }
    cta_first[n] = (int16_t)first;
    return first;
}

static int grad_job_cost(int na, int kind, int loss_mode) {
    if (loss_mode == RCMARL_LOSS_CE) return grad_row_cost(2 * na, NACT);
    return grad_row_cost(kind == RCMARL_IN_SA ? 3 * na : 2 * na, 1);
}

// host copy of TileLayout<DIN, NOUT> behind rcmarl_grad_tile_map
template <int DIN, int NOUT>
static int grad_tile_map(int32_t* info, int32_t* params, int64_t cap) {
    using L = TileLayout<DIN, NOUT>;
    info[0] = L::NT; info[1] = L::TA; info[2] = L::TD; info[3] = L::NG; info[4] = L::PH2_FFMA;
    info[5] = L::L3T ? param_count(DIN, NOUT) : off_W3(DIN);
    if (cap < (int64_t)L::NT * L::NACC) return RCMARL_ERR_ARG;
    for (int t = 0; t < L::NT; ++t)
        for (int e = 0; e < L::NACC; ++e) params[t * L::NACC + e] = L::tile_param(t, e / L::TD, e % L::TD);
    return RCMARL_OK;
}



template <int NA>
static int launch_mb_persist(const MbParams& P, int n_ctas, cudaStream_t st) {
    constexpr int NW = grad_warps<NA, RCMARL_LOSS_MSE>();
    constexpr size_t smem = grad_smem_bytes<NA, RCMARL_LOSS_MSE>();
    static int resident = -1;                          // CTAs that can be co-resident (the cells protocol needs all of them)
    if (resident < 0) {
        if (set_smem(mb_persist_kernel<NA>, smem)) return RCMARL_ERR_CUDA;
        int per_sm = 0;
        RC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mb_persist_kernel<NA>, 32 * NW, smem));
        resident = per_sm * sm_count_cached();
    }
    if (n_ctas > resident) return RCMARL_ERR_ARG;
    return launch_pdl(mb_persist_kernel<NA>, dim3(n_ctas), dim3(32 * NW), smem, st, P);
}

// [first, last) byte range, never empty
struct Range {
    uintptr_t first, last;
};

static bool overlap(const Range& a, const Range& b) { return a.first < b.last && b.first < a.last; }

// up to CAP byte ranges
template <int CAP>
struct RangeList {
    Range at[CAP];
    int n = 0;
    // n_bytes bytes at p
    void bytes(const void* p, int64_t n_bytes) { at[n++] = {(uintptr_t)p, (uintptr_t)p + (uintptr_t)n_bytes}; }
    // n_floats floats at p
    void floats(const float* p, int64_t n_floats) { row(p, 0, 0, n_floats); }
    // n_floats floats at base + r * stride floats
    void row(const float* base, int64_t r, int64_t stride, int64_t n_floats) {
        const uintptr_t first = (uintptr_t)base + (uintptr_t)(r * stride * (int64_t)sizeof(float));
        at[n++] = {first, first + (uintptr_t)(n_floats * (int64_t)sizeof(float))};
    }
    // the rows r < n_rows
    void rows(const float* base, int n_rows, int64_t stride, int64_t n_floats) {
        for (int r = 0; r < n_rows; ++r) row(base, r, stride, n_floats);
    }
    // the rows nodes[k], k < n_nodes, except the crafted slots (-1)
    void nodes(const float* base, const int32_t* nodes, int n_nodes, int64_t stride, int64_t n_floats) {
        for (int k = 0; k < n_nodes; ++k)
            if (nodes[k] >= 0) row(base, nodes[k], stride, n_floats);
    }
};

// What the CTAs of one launch write (w) and read (r).  A CTA may read its inputs before it writes, but the CTAs of
// other jobs run concurrently: a launch is refused when a written range overlaps another written range or a read range
// of any job of the launch.  Read ranges may overlap each other.  Sized for the most ranges of one launch: the 2 x 16
// written rows per job of rcmarl_momentum_mix and the 2 x 16 + 1 read ranges per job of rcmarl_history_attack.
struct RangeSet {
    RangeList<2 * RCMARL_MAX_JOBS * RCMARL_MAX_NEIGHBOURS> w;
    RangeList<RCMARL_MAX_JOBS * (2 * RCMARL_MAX_NEIGHBOURS + 1)> r;
    // Sorts the written ranges by start, so the check takes O((w.n + r.n) log w.n) comparisons instead of one per pair.
    bool overlaps() {
        Range* const w0 = w.at;
        Range* const w1 = w.at + w.n;
        std::sort(w0, w1, [](const Range& a, const Range& b) {
            return a.first < b.first || (a.first == b.first && a.last < b.last);
        });
        for (const Range* a = w0; a + 1 < w1; ++a)
            if (a->last > a[1].first) return true;
        // the written ranges are now disjoint and sorted by start, hence by end too: of them only the first one that
        // ends after a read range's start can overlap it
        for (int k = 0; k < r.n; ++k) {
            const Range* it =
                std::upper_bound(w0, w1, r.at[k].first, [](uintptr_t x, const Range& q) { return x < q.last; });
            if (it != w1 && it->first < r.at[k].last) return true;
        }
        return false;
    }
};

// One CTA of `threads` per job, staging up to `floats` floats (the largest job's) in dynamic shared memory.  The kernel
// also has static shared memory, so the default 48 KB limit applies to static + dynamic: its limit is lifted to the
// staging bound of `bound` floats once per device, before the kernel's first launch there (opted: the flags of this
// Kernel), independent of any other launch.
template <auto Kernel, typename Params>
static int launch_staged(const Params& P, int n_jobs, int bound, int64_t floats, int threads, void* stream) {
    static bool opted[64] = {};
    int dev = 0;
    RC_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !opted[dev]) {
        RC_CUDA(cudaFuncSetAttribute((const void*)Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(sizeof(float) * bound)));
        if (dev >= 0 && dev < 64) opted[dev] = true;
    }
    Kernel<<<n_jobs, threads, sizeof(float) * (size_t)floats, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

}  // namespace rcmarl

using namespace rcmarl;

extern "C" {

int64_t rcmarl_workspace_bytes(int n_jobs, int max_params) {
    if (n_jobs < 1) n_jobs = 1;
    const int64_t ctas = (int64_t)sm_count_cached() * 2 + 2 * (int64_t)n_jobs;
    return ctas * (int64_t)(max_params + 1) * (int64_t)sizeof(float);
}

int rcmarl_grad_grid_plan(int n_agents, const int32_t* kinds_host, int n_jobs, int loss_mode, int64_t n_rows, int balanced,
                          int sm_count, int32_t* ctas_host) {
    if ((n_agents != 5 && n_agents != 16) || !kinds_host || !ctas_host || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS ||
        n_rows < 0 || sm_count < 1 || (loss_mode != RCMARL_LOSS_MSE && loss_mode != RCMARL_LOSS_CE))
        return RCMARL_ERR_ARG;
    int cost[RCMARL_MAX_JOBS], g[RCMARL_MAX_JOBS];
    for (int j = 0; j < n_jobs; ++j) {
        if (kinds_host[j] < 0 || kinds_host[j] > 2) return RCMARL_ERR_ARG;
        cost[j] = grad_job_cost(n_agents, kinds_host[j], loss_mode);
    }
    const bool ce = loss_mode == RCMARL_LOSS_CE;
    const int cpc = n_agents == 5 ? (ce ? grad_warps<5, RCMARL_LOSS_CE>() : grad_warps<5, RCMARL_LOSS_MSE>())
                                  : (ce ? grad_warps<16, RCMARL_LOSS_CE>() : grad_warps<16, RCMARL_LOSS_MSE>());
    plan_shares(n_jobs, cost, (n_rows + 63) / 64, cpc, sm_count, balanced != 0, g);
    for (int j = 0; j < n_jobs; ++j) ctas_host[j] = g[j];
    return RCMARL_OK;
}

int rcmarl_grad_tile_map(int d_in, int n_out, int32_t* info, int32_t* params, int64_t cap) {
    if (!info || !params) return RCMARL_ERR_ARG;
    if (n_out == 1) {
        if (d_in == 10) return grad_tile_map<10, 1>(info, params, cap);
        if (d_in == 15) return grad_tile_map<15, 1>(info, params, cap);
        if (d_in == 32) return grad_tile_map<32, 1>(info, params, cap);
        if (d_in == 48) return grad_tile_map<48, 1>(info, params, cap);
    } else if (n_out == NACT) {
        if (d_in == 10) return grad_tile_map<10, NACT>(info, params, cap);
        if (d_in == 32) return grad_tile_map<32, NACT>(info, params, cap);
    }
    return RCMARL_ERR_ARG;
}

int rcmarl_values(const rcmarl_rows* rows, const rcmarl_value_job* jobs, int n_jobs, void* stream) {
    if (int e = check_rows(rows)) return e;
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    if (rows->n_rows == 0) return RCMARL_OK;
    ValuesParams P;
    P.rows = *rows;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_value_job& q = jobs[j];
        if (!q.out || q.n_terms < 1 || q.n_terms > RCMARL_MAX_TERMS) return RCMARL_ERR_ARG;
        if (q.n_out != 1 && !(q.n_out == NACT && q.n_terms == 1 && q.kind[0] != RCMARL_IN_SA)) return RCMARL_ERR_ARG;
        for (int t = 0; t < q.n_terms; ++t)
            if (!q.w[t] || q.kind[t] < 0 || q.kind[t] > 2) return RCMARL_ERR_ARG;
        P.jobs[j] = q;
    }
    cudaStream_t st = (cudaStream_t)stream;
    return rows->n_agents == 5 ? launch_values<5>(P, n_jobs, st) : launch_values<16>(P, n_jobs, st);
}

int rcmarl_grad(const rcmarl_rows* rows, const rcmarl_grad_job* jobs, int n_jobs, int loss_mode, void* ws,
                int64_t ws_bytes, void* stream) {
    if (int e = check_rows(rows)) return e;
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS || !ws) return RCMARL_ERR_ARG;
    if (loss_mode != RCMARL_LOSS_MSE && loss_mode != RCMARL_LOSS_CE) return RCMARL_ERR_ARG;
    const int NA = rows->n_agents;
    GradParams P;
    ReduceParams Q;
    P.rows = *rows;
    int maxn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_grad_job& q = jobs[j];
        if (!q.w || !q.target || !q.sums || q.kind < 0 || q.kind > 2 || q.target_stride < 1) return RCMARL_ERR_ARG;
        if (q.time_idx && !rows->time_idx) return RCMARL_ERR_ARG;   /* overrides need the gathered row mode */
        if (loss_mode == RCMARL_LOSS_CE && (q.kind != RCMARL_IN_S || q.action_agent < 0 || q.action_agent >= NA))
            return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        const int n = loss_mode == RCMARL_LOSS_CE ? param_count(2 * NA, NACT)
                                                   : param_count(q.kind == RCMARL_IN_SA ? 3 * NA : 2 * NA, 1);
        Q.sums[j] = q.sums;
        Q.n[j] = n + 1;
        if (n + 1 > maxn) maxn = n + 1;
    }
    // CTA shares by cost; each warp of a CTA takes one 64-row chunk per sweep
    int cost[RCMARL_MAX_JOBS];
    for (int j = 0; j < n_jobs; ++j) cost[j] = grad_job_cost(NA, jobs[j].kind, loss_mode);
    const bool ce = loss_mode == RCMARL_LOSS_CE;
    const int cpc = NA == 5 ? (ce ? grad_warps<5, RCMARL_LOSS_CE>() : grad_warps<5, RCMARL_LOSS_MSE>())
                            : (ce ? grad_warps<16, RCMARL_LOSS_CE>() : grad_warps<16, RCMARL_LOSS_MSE>());
    P.partial = (float*)ws;
    P.n_jobs = n_jobs;
    P.stride = maxn;
    const int n_ctas = plan_grid(n_jobs, cost, (rows->n_rows + 63) / 64, cpc, true, P.cta_first);
    if ((int64_t)n_ctas * maxn * (int64_t)sizeof(float) > ws_bytes) return RCMARL_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int e = NA == 5 ? (ce ? launch_grad<5, RCMARL_LOSS_CE>(P, n_ctas, st) : launch_grad<5, RCMARL_LOSS_MSE>(P, n_ctas, st))
                          : (ce ? launch_grad<16, RCMARL_LOSS_CE>(P, n_ctas, st) : launch_grad<16, RCMARL_LOSS_MSE>(P, n_ctas, st));
    if (e) return e;
    Q.partial = (const float*)ws;
    Q.slots.step = 1;
    Q.slots.stride = maxn;
    for (int j = 0; j < n_jobs; ++j) {
        Q.slots.first[j] = P.cta_first[j];
        Q.slots.count[j] = P.cta_first[j + 1] - P.cta_first[j];
    }
    return reduce_partials(Q, n_jobs, maxn, st);
}

int64_t rcmarl_minibatch_cells_bytes(int n_jobs, int max_params) {
    if (n_jobs < 1) n_jobs = 1;
    // level 1: one row of cells per CTA (<= SMs); level 2 (single GPU): 2 slots x n_jobs rows; + the error word
    // (sized generously: a row per CTA AND chain)
    return ((int64_t)sm_count_cached() * (int64_t)n_jobs + 2 * (int64_t)n_jobs) * (int64_t)(max_params + 1) * (int64_t)sizeof(uint2) + 64;
}

int64_t rcmarl_minibatch_steps(int epochs, int n_times, int mb_times) {
    if (epochs < 1 || n_times < 1 || mb_times < 1) return 0;
    return (int64_t)epochs * ((n_times + mb_times - 1) / mb_times);
}

int rcmarl_minibatch_fit(const rcmarl_rows* rows, const rcmarl_grad_job* gjobs, const rcmarl_sgd_job* sjobs, int n_jobs,
                         int epochs, int n_times, int mb_times, float lr, void* cells, int64_t cells_bytes,
                         uint32_t seq_first, void* stream) {
    if (!rows) return RCMARL_ERR_ARG;
    MbParams P;
    P.rows = *rows;
    P.rows.n_rows = 0;
    P.rows.time_idx = nullptr;
    if (int e = check_rows(&P.rows)) return e;
    if (!gjobs || !sjobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS || !cells || epochs < 1 || n_times < 1 || mb_times < 1 ||
        seq_first < 1)
        return RCMARL_ERR_ARG;
    const int NA = rows->n_agents;
    int maxn = 0;
    int cost[RCMARL_MAX_JOBS];
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_grad_job& q = gjobs[j];
        if (!q.w || !q.target || !q.time_idx || q.kind < 0 || q.kind > 2 || q.target_stride < 1) return RCMARL_ERR_ARG;
        if (!sjobs[j].dst || sjobs[j].dst != sjobs[j].src || (const float*)sjobs[j].dst != q.w) return RCMARL_ERR_ARG;
        const int n = param_count(q.kind == RCMARL_IN_SA ? 3 * NA : 2 * NA, 1);
        if (sjobs[j].n != n || sjobs[j].first != 0) return RCMARL_ERR_ARG;
        MbChain& c = P.chains[j];
        c.w = sjobs[j].dst; c.target = q.target; c.time_idx = q.time_idx; c.loss_out = sjobs[j].loss_out;
        c.target_stride = q.target_stride; c.lr = sjobs[j].coef > 0.f ? sjobs[j].coef : lr;
        c.loss_coef = sjobs[j].loss_coef; c.kind = q.kind; c.loss_accumulate = sjobs[j].loss_accumulate;
        cost[j] = grad_job_cost(NA, q.kind, RCMARL_LOSS_MSE);
        if (n + 1 > maxn) maxn = n + 1;
    }
    const int cpc = NA == 5 ? grad_warps<5, RCMARL_LOSS_MSE>() : grad_warps<16, RCMARL_LOSS_MSE>();
    const int64_t n_rows_mb = (int64_t)(n_times < mb_times ? n_times : mb_times) * rows->n_envs;
    // CTA shares by cost, as in rcmarl_grad.  A mapping with every
    // CTA serving every chain in turn (reduction of a chain hidden behind the other chains' turns) was measured
    // slower and removed.
    const int n_ctas = plan_grid(n_jobs, cost, (n_rows_mb + 63) / 64, cpc, true, P.cta_first);
    P.n_chains = n_jobs; P.epochs = epochs; P.n_times = n_times; P.mb_times = mb_times; P.stride = maxn;
    const int64_t steps = rcmarl_minibatch_steps(epochs, n_times, mb_times);
    if ((uint64_t)seq_first + (uint64_t)steps >= 0xFFFFFFFFull) return RCMARL_ERR_ARG;
    const int64_t l1 = (int64_t)n_ctas * maxn, l2 = 2 * (int64_t)n_jobs * maxn;
    if ((l1 + l2) * (int64_t)sizeof(uint2) + 64 > cells_bytes) return RCMARL_ERR_WORKSPACE;
    if (((uintptr_t)cells & 15) != 0) return RCMARL_ERR_ARG;
    P.cells1 = (uint2*)cells;
    P.seq1 = seq_first;
    if (comm_bound()) {
        if (!comm_reserve(&P.comm, (int64_t)n_jobs * maxn, (uint32_t)steps)) return RCMARL_ERR_ARG;
    } else {
        for (int p = 0; p < COMM_MAX_WORLD; ++p) P.comm.cells[p] = nullptr;
        P.comm.cells[0] = (uint2*)cells + l1;
        P.comm.error = (uint32_t*)((uint2*)cells + l1 + l2);
        P.comm.max_floats = (int64_t)n_jobs * maxn;
        P.comm.rank = 0; P.comm.world = 1; P.comm.seq = seq_first;
    }
    cudaStream_t st = (cudaStream_t)stream;
    return NA == 5 ? launch_mb_persist<5>(P, n_ctas, st) : launch_mb_persist<16>(P, n_ctas, st);
}

// an unknown rcmarl_agg_rule, or TRIM with fewer than 2H + 1 values (callers have checked 0 <= H < n_in)
static bool bad_rule(int rule, int H, int n_in) {
    return rule < RCMARL_AGG_CLIP || rule > RCMARL_AGG_WMSR || (rule == RCMARL_AGG_TRIM && 2 * H >= n_in);
}

// a receiver's rule: a known family and rule, and an H that rule allows for n_rows messages (COORD: the checks of
// rcmarl_consensus_hidden)
static bool bad_receiver_rule(int family, int rule, int H, int n_rows) {
    if (H < 0 || H >= n_rows) return true;
    if (family == RCMARL_TAILOR_COORD) return bad_rule(rule, H, n_rows);
    if (family == RCMARL_TAILOR_SPECTRAL) return rule != RCMARL_SPECTRAL_DNC;
    if (family != RCMARL_TAILOR_VECTOR || rule < RCMARL_VEC_KRUM || rule > RCMARL_VEC_GMED) return true;
    return (rule == RCMARL_VEC_KRUM || rule == RCMARL_VEC_MKRUM) && n_rows < H + 3;
}

// a negative row among the first n of a node list (in-nodes or honest rows; callers have checked n)
static bool bad_nodes(const int32_t* nodes, int n) {
    for (int k = 0; k < n; ++k)
        if (nodes[k] < 0) return true;
    return false;
}

int rcmarl_team(const rcmarl_rows* rows, const rcmarl_team_job* jobs, int n_jobs, void* ws, int64_t ws_bytes,
                void* stream) {
    if (int e = check_rows(rows)) return e;
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    const int NA = rows->n_agents;
    TeamParams P;
    ReduceParams Q;
    P.rows = *rows;
    bool any_sums = false;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_team_job& q = jobs[j];
        if (!q.w || q.kind < 0 || q.kind > 2) return RCMARL_ERR_ARG;
        if (!q.agg_in) {
            if (!q.msgs || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS || q.H < 0 || q.H >= q.n_in) return RCMARL_ERR_ARG;
            if (bad_nodes(q.in_nodes, q.n_in) || bad_rule(q.rule, q.H, q.n_in)) return RCMARL_ERR_ARG;
        }
        if (!q.sums && !q.agg_out) return RCMARL_ERR_ARG;
        any_sums |= (q.sums != nullptr);
        P.jobs[j] = q;
        if (q.agg_in) P.jobs[j].n_in = 0;         // the aggregate is supplied: no neighbour head is staged or read
        Q.sums[j] = q.sums;
        Q.n[j] = q.sums ? TEAM_N : 0;
    }
    // one launch per input kind (see TeamParams::job_list); each fills the GPU on its own: 128 threads x 2 rows, 3 CTAs / SM
    int gy_of[RCMARL_MAX_JOBS], gy_max = 0;
    int lists[2][RCMARL_MAX_JOBS], n_list[2] = {0, 0};
    for (int j = 0; j < n_jobs; ++j) {
        const int g = jobs[j].kind == RCMARL_IN_SA ? 0 : 1;
        lists[g][n_list[g]++] = j;
    }
    for (int g = 0; g < 2; ++g) {
        if (!n_list[g]) continue;
        const int gy = grid_y_for((rows->n_rows + 255) / 256, n_list[g], 3);
        for (int k = 0; k < n_list[g]; ++k) gy_of[lists[g][k]] = gy;
        gy_max = gy > gy_max ? gy : gy_max;
    }
    if (any_sums) {
        if (!ws || (int64_t)gy_max * n_jobs * TEAM_N * (int64_t)sizeof(float) > ws_bytes) return RCMARL_ERR_WORKSPACE;
    }
    P.partial = (float*)ws;
    P.n_jobs = n_jobs;
    P.stride = TEAM_N;
    cudaStream_t st = (cudaStream_t)stream;
    for (int g = 0; g < 2; ++g) {
        if (!n_list[g]) continue;
        for (int k = 0; k < n_list[g]; ++k) P.job_list[k] = lists[g][k];
        const int gy = gy_of[lists[g][0]];
        const int e = NA == 5 ? launch_team<5>(P, n_list[g], gy, st) : launch_team<16>(P, n_list[g], gy, st);
        if (e) return e;
    }
    if (!any_sums) return RCMARL_OK;
    Q.partial = (const float*)ws;
    Q.slots.step = n_jobs;                        // team_kernel writes its partials [y][job] interleaved
    Q.slots.stride = TEAM_N;
    for (int j = 0; j < n_jobs; ++j) { Q.slots.first[j] = j; Q.slots.count[j] = gy_of[j]; }
    return reduce_partials(Q, n_jobs, TEAM_N, st);
}

int rcmarl_consensus_hidden(const rcmarl_consensus_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    ConsensusParams P;
    int maxn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_consensus_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS || q.H < 0 || q.H >= q.n_in || q.n_hidden < 1)
            return RCMARL_ERR_ARG;
        if (bad_nodes(q.in_nodes, q.n_in) || bad_rule(q.rule, q.H, q.n_in)) return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        if (q.n_hidden > maxn) maxn = q.n_hidden;
    }
    consensus_hidden_kernel<<<dim3((maxn + 255) / 256, n_jobs), 256, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_attack(const rcmarl_attack_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    AttackParams P;
    int maxn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_attack_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_honest < 1 || q.n_honest > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (bad_nodes(q.honest, q.n_honest)) return RCMARL_ERR_ARG;
        if (q.kind < RCMARL_ATTACK_ALIE || q.kind > RCMARL_ATTACK_GAUSS || !std::isfinite(q.param)) return RCMARL_ERR_ARG;
        if (q.kind == RCMARL_ATTACK_GAUSS && q.param < 0.f) return RCMARL_ERR_ARG;
        if (q.attacker > 255u || q.receiver > 255u) return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        if (q.n > maxn) maxn = q.n;
    }
    attack_kernel<<<dim3((maxn + 255) / 256, n_jobs), 256, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_vector_aggregate(const rcmarl_vector_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    VectorParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_vector_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (bad_receiver_rule(RCMARL_TAILOR_VECTOR, q.rule, q.H, q.n_in) || bad_nodes(q.in_nodes, q.n_in))
            return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)(q.n_in + 1) * q.n;
        if (floats > RCMARL_VECTOR_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst and weights_out, reads the in-node rows
        S.w.floats(q.dst, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<vector_agg_kernel>(P, n_jobs, RCMARL_VECTOR_MAX_FLOATS, max_floats, VEC_THREADS, stream);
}

int rcmarl_dnc_aggregate(const rcmarl_vector_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    VectorParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_vector_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (bad_receiver_rule(RCMARL_TAILOR_SPECTRAL, q.rule, q.H, q.n_in) || bad_nodes(q.in_nodes, q.n_in))
            return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)(q.n_in + 2) * q.n;
        if (floats > RCMARL_DNC_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst and weights_out, reads the in-node rows
        S.w.floats(q.dst, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<dnc_agg_kernel>(P, n_jobs, RCMARL_DNC_MAX_FLOATS, max_floats, VEC_THREADS, stream);
}

int rcmarl_subset_aggregate(const rcmarl_vector_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    VectorParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_vector_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if ((q.rule != RCMARL_SUBSET_MDA && q.rule != RCMARL_SUBSET_SMEA) || q.H < 0 || q.H >= q.n_in) return RCMARL_ERR_ARG;
        if (bad_nodes(q.in_nodes, q.n_in)) return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)q.n_in * q.n;
        if (floats > RCMARL_SUBSET_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst and weights_out, reads the in-node rows
        S.w.floats(q.dst, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<subset_agg_kernel>(P, n_jobs, RCMARL_SUBSET_MAX_FLOATS, max_floats, VEC_THREADS, stream);
}

int rcmarl_ios_aggregate(const rcmarl_vector_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    VectorParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_vector_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (q.rule != RCMARL_FILTER_IOS || q.H < 0 || q.H >= q.n_in || bad_nodes(q.in_nodes, q.n_in)) return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)(q.n_in + 2) * q.n;
        if (floats > RCMARL_IOS_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst and weights_out, reads the in-node rows
        S.w.floats(q.dst, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<ios_agg_kernel>(P, n_jobs, RCMARL_IOS_MAX_FLOATS, max_floats, VEC_THREADS, stream);
}

int rcmarl_nnm_mix(const rcmarl_vector_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    VectorParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_vector_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (q.rule != RCMARL_MIX_NNM || q.H < 0 || q.H >= q.n_in) return RCMARL_ERR_ARG;
        if (bad_nodes(q.in_nodes, q.n_in)) return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)q.n_in * q.n;
        if (floats > RCMARL_NNM_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes the n_in dst rows and the n_in^2 weights, reads the in-node rows
        S.w.rows(q.dst, q.n_in, q.msg_stride, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, (int64_t)q.n_in * q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<nnm_mix_kernel>(P, n_jobs, RCMARL_NNM_MAX_FLOATS, max_floats, VEC_THREADS, stream);
}

int rcmarl_arc_clip(const rcmarl_vector_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    VectorParams P;
    RangeSet S;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_vector_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (q.rule != RCMARL_MIX_ARC || q.H < 0 || q.H >= q.n_in) return RCMARL_ERR_ARG;
        if (bad_nodes(q.in_nodes, q.n_in)) return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        // writes the n_in dst rows and the n_in factors, reads the in-node rows
        S.w.rows(q.dst, q.n_in, q.msg_stride, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    arc_clip_kernel<<<n_jobs, VEC_THREADS, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_bucket_mix(const rcmarl_bucket_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    BucketParams P;
    RangeSet S;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_bucket_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (bad_nodes(q.in_nodes, q.n_in) || q.s < 1 || q.net > 1u || q.receiver > 255u) return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        // writes the n_out = 1 + ceil((n_in - 1) / s) dst rows and the n_out * n_in weights, reads the in-node rows
        const int n_out = q.n_in == 1 ? 1 : 1 + (q.n_in - 2) / q.s + 1;
        S.w.rows(q.dst, n_out, q.msg_stride, q.n);
        if (q.weights_out) S.w.floats(q.weights_out, (int64_t)n_out * q.n_in);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    bucket_mix_kernel<<<n_jobs, VEC_THREADS, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_momentum_mix(const rcmarl_momentum_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    MomentumParams P;
    RangeSet S;
    int maxn = 0, max_in = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_momentum_job& q = jobs[j];
        if (!q.dst || !q.msgs || !q.ref || !q.momentum || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS)
            return RCMARL_ERR_ARG;
        if (bad_nodes(q.in_nodes, q.n_in)) return RCMARL_ERR_ARG;
        if (!std::isfinite(q.beta) || q.beta < 0.f || q.beta >= 1.f || (q.first != 0 && q.first != 1))
            return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        if (q.n > maxn) maxn = q.n;
        if (q.n_in > max_in) max_in = q.n_in;
        // writes the dst rows and the M rows, reads the in-node rows and (below) the ref
        S.w.rows(q.dst, q.n_in, q.msg_stride, q.n);
        S.w.rows(q.momentum, q.n_in, q.momentum_stride, q.n);
        S.r.nodes(q.msgs, q.in_nodes, q.n_in, q.msg_stride, q.n);
    }
    // and no ref may overlap an in-node row of any job of the launch (two refs may coincide)
    const int n_rows = S.r.n;
    for (int j = 0; j < n_jobs; ++j) S.r.floats(jobs[j].ref, jobs[j].n);
    for (int c = n_rows; c < S.r.n; ++c)
        for (int k = 0; k < n_rows; ++k)
            if (overlap(S.r.at[c], S.r.at[k])) return RCMARL_ERR_ARG;
    if (S.overlaps()) return RCMARL_ERR_ARG;
    momentum_mix_kernel<<<dim3((maxn + 255) / 256, n_jobs, max_in), 256, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_adaptive_attack(const rcmarl_adaptive_attack_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    AdaptiveParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_adaptive_attack_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_honest < 1 || q.n_honest > RCMARL_MAX_NEIGHBOURS) return RCMARL_ERR_ARG;
        if (bad_nodes(q.honest, q.n_honest)) return RCMARL_ERR_ARG;
        if (q.kind < RCMARL_ADAPT_MINMAX || q.kind > RCMARL_ADAPT_MINSUM || q.dev < RCMARL_DEV_UV || q.dev > RCMARL_DEV_SGN)
            return RCMARL_ERR_ARG;
        if (!std::isfinite(q.scale) || q.scale < 0.f) return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)(q.n_honest + 2) * q.n;
        if (floats > RCMARL_ADAPTIVE_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst and gamma_out, reads the honest rows
        S.w.floats(q.dst, q.n);
        if (q.gamma_out) S.w.floats(q.gamma_out, 1);
        S.r.nodes(q.msgs, q.honest, q.n_honest, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<adaptive_attack_kernel>(P, n_jobs, RCMARL_ADAPTIVE_MAX_FLOATS, max_floats, ADA_THREADS,
                                                 stream);
}

// the slot list, direction and scale of a tailored job (everything but its rule); n_real receives its real slots
static bool bad_tailored_slots(const rcmarl_tailored_attack_job& q, int& n_real) {
    if (!q.dst || !q.msgs || q.n < 1 || q.n_in < 1 || q.n_in > RCMARL_MAX_NEIGHBOURS) return true;
    if (q.honest_mask >> q.n_in) return true;                        // a bit past the slot list
    n_real = 0;
    for (int k = 0; k < q.n_in; ++k) {
        if (q.slots[k] < -1) return true;
        if (q.slots[k] == -1 && ((q.honest_mask >> k) & 1u)) return true;   // a crafted slot marked honest
        n_real += q.slots[k] >= 0 ? 1 : 0;
    }
    if (n_real == q.n_in || q.honest_mask == 0u) return true;        // no crafted slot, no honest slot
    if (q.dev < RCMARL_DEV_UV || q.dev > RCMARL_DEV_SGN) return true;
    return !std::isfinite(q.scale) || q.scale < 0.f;
}

int rcmarl_tailored_attack(const rcmarl_tailored_attack_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    TailoredParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_tailored_attack_job& q = jobs[j];
        int n_real = 0;
        if (bad_tailored_slots(q, n_real)) return RCMARL_ERR_ARG;
        if (q.family == RCMARL_TAILOR_SPECTRAL || bad_receiver_rule(q.family, q.rule, q.H, q.n_in)) return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)(q.n_in + 3) * q.n;
        if (floats > RCMARL_TAILORED_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst and gamma_out, reads the real slots' rows
        S.w.floats(q.dst, q.n);
        if (q.gamma_out) S.w.floats(q.gamma_out, 1);
        S.r.nodes(q.msgs, q.slots, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<tailored_attack_kernel>(P, n_jobs, RCMARL_TAILORED_MAX_FLOATS, max_floats, ADA_THREADS,
                                                 stream);
}

}  // extern "C"

// ARC's staging in an ARC form of the pipeline or history search: k_clip rows, and slot 0 (the receiver's own) real
static bool arc_staging(const rcmarl_tailored_attack_job& q, bool arc, int64_t& floats) {
    if (!arc) return false;
    floats += (int64_t)(2 * q.H * (q.n_in - q.H) / q.n_in) * q.n;
    return q.slots[0] < 0;
}

// the receiver's rule in a subset form of the pipeline or history search: family SUBSET, MDA or SMEA, 0 <= H < n_rows
static bool bad_subset_receiver(int family, int rule, int H, int n_rows) {
    return family != RCMARL_TAILOR_SUBSET || (rule != RCMARL_SUBSET_MDA && rule != RCMARL_SUBSET_SMEA) || H < 0 ||
           H >= n_rows;
}

// the receiver's rule in an IOS form of the pipeline or history search: family FILTER, IOS, 0 <= H < n_rows
static bool bad_ios_receiver(int family, int rule, int H, int n_rows) {
    return family != RCMARL_TAILOR_FILTER || rule != RCMARL_FILTER_IOS || H < 0 || H >= n_rows;
}

// the receiver's rule for the rule stage STAGE of the pipeline or history search
template <int STAGE>
static bool bad_stage_receiver(int family, int rule, int H, int n_rows) {
    if (STAGE == STAGE_SUBSET) return bad_subset_receiver(family, rule, H, n_rows);
    if (STAGE == STAGE_IOS) return bad_ios_receiver(family, rule, H, n_rows);
    return bad_receiver_rule(family, rule, H, n_rows);
}

template <bool ARC, int STAGE>
static int pipeline_attack(const rcmarl_pipeline_attack_job* jobs, int n_jobs, void* stream) {
    constexpr int bound = STAGE == STAGE_SUBSET ? RCMARL_SUBSET_ATTACK_MAX_FLOATS : RCMARL_PIPELINE_MAX_FLOATS;
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    PipelineParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_pipeline_attack_job& pj = jobs[j];
        const rcmarl_tailored_attack_job& q = pj.attack;
        int n_real = 0;
        if (bad_tailored_slots(q, n_real)) return RCMARL_ERR_ARG;
        int n_rows = q.n_in, n_mixed = 0;
        if (pj.mixing == RCMARL_PIPE_NNM) {
            n_mixed = q.n_in;
        } else if (pj.mixing == RCMARL_PIPE_BUCKET) {
            if (pj.s < 1 || pj.n_perms < 1 || pj.n_perms > RCMARL_PIPELINE_MAX_PERMS) return RCMARL_ERR_ARG;
            if (pj.attacker > 255u || pj.receiver > 255u || pj.net > 1u) return RCMARL_ERR_ARG;
            n_rows = 1 + (q.n_in - 2) / pj.s + 1;                    // n_in >= 2: a crafted and an honest slot
            n_mixed = n_rows - 1;
        } else if (pj.mixing != RCMARL_PIPE_NONE) {
            return RCMARL_ERR_ARG;
        }
        if (bad_stage_receiver<STAGE>(q.family, q.rule, q.H, n_rows)) return RCMARL_ERR_ARG;
        // DnC's mean and IOS's centre: n doubles in front of the real slots
        const bool f64 = q.family == RCMARL_TAILOR_SPECTRAL || q.family == RCMARL_TAILOR_FILTER;
        int64_t floats = (int64_t)(n_real + n_mixed + 4 + (f64 ? 2 : 0)) * q.n;
        if (arc_staging(q, ARC, floats) || floats > bound) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = pj;
        // writes dst, gamma_out and model_out, reads the real slots' rows
        S.w.floats(q.dst, q.n);
        if (q.gamma_out) S.w.floats(q.gamma_out, 1);
        if (pj.model_out) S.w.floats(pj.model_out, q.n);
        S.r.nodes(q.msgs, q.slots, q.n_in, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<pipeline_attack_kernel<ARC, STAGE>>(P, n_jobs, bound, max_floats, ADA_THREADS, stream);
}

template <bool ARC, int STAGE>
static int history_attack(const rcmarl_history_attack_job* jobs, int n_jobs, void* stream) {
    constexpr int bound = STAGE == STAGE_SUBSET ? RCMARL_SUBSET_ATTACK_MAX_FLOATS : RCMARL_HISTORY_MAX_FLOATS;
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    HistoryParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_history_attack_job& hj = jobs[j];
        const rcmarl_tailored_attack_job& q = hj.attack;
        int n_real = 0;
        if (bad_tailored_slots(q, n_real)) return RCMARL_ERR_ARG;
        if (bad_stage_receiver<STAGE>(q.family, q.rule, q.H, q.n_in)) return RCMARL_ERR_ARG;
        if (!hj.ref || !hj.momentum) return RCMARL_ERR_ARG;
        if (!std::isfinite(hj.beta) || hj.beta < 0.f || hj.beta >= 1.f || (hj.first != 0 && hj.first != 1))
            return RCMARL_ERR_ARG;
        if (hj.own_mask == 0u || (hj.own_mask >> q.n_in)) return RCMARL_ERR_ARG;
        for (int k = 0; k < q.n_in; ++k)
            if (((hj.own_mask >> k) & 1u) && q.slots[k] >= 0) return RCMARL_ERR_ARG;   // an own bit on a real slot
        const bool f64 = q.family == RCMARL_TAILOR_SPECTRAL || q.family == RCMARL_TAILOR_FILTER;
        int64_t floats = (int64_t)(q.n_in + 4 + (f64 ? 2 : 0)) * q.n;
        if (arc_staging(q, ARC, floats) || floats > bound) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = hj;
        // writes dst, gamma_out and model_out, reads the real slots' rows, the ref and the n_in M rows
        S.w.floats(q.dst, q.n);
        if (q.gamma_out) S.w.floats(q.gamma_out, 1);
        if (hj.model_out) S.w.floats(hj.model_out, q.n);
        S.r.nodes(q.msgs, q.slots, q.n_in, q.msg_stride, q.n);
        S.r.floats(hj.ref, q.n);
        S.r.rows(hj.momentum, q.n_in, hj.momentum_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<history_attack_kernel<ARC, STAGE>>(P, n_jobs, bound, max_floats, ADA_THREADS, stream);
}

extern "C" {

int rcmarl_pipeline_attack(const rcmarl_pipeline_attack_job* jobs, int n_jobs, void* stream) {
    return pipeline_attack<false, STAGE_BASE>(jobs, n_jobs, stream);
}

int rcmarl_pipeline_arc_attack(const rcmarl_pipeline_attack_job* jobs, int n_jobs, void* stream) {
    return pipeline_attack<true, STAGE_BASE>(jobs, n_jobs, stream);
}

int rcmarl_history_attack(const rcmarl_history_attack_job* jobs, int n_jobs, void* stream) {
    return history_attack<false, STAGE_BASE>(jobs, n_jobs, stream);
}

int rcmarl_history_arc_attack(const rcmarl_history_attack_job* jobs, int n_jobs, void* stream) {
    return history_attack<true, STAGE_BASE>(jobs, n_jobs, stream);
}

int rcmarl_subset_pipeline_attack(const rcmarl_pipeline_attack_job* jobs, int n_jobs, int arc, void* stream) {
    if (arc != 0 && arc != 1) return RCMARL_ERR_ARG;
    return arc ? pipeline_attack<true, STAGE_SUBSET>(jobs, n_jobs, stream)
               : pipeline_attack<false, STAGE_SUBSET>(jobs, n_jobs, stream);
}

int rcmarl_subset_history_attack(const rcmarl_history_attack_job* jobs, int n_jobs, int arc, void* stream) {
    if (arc != 0 && arc != 1) return RCMARL_ERR_ARG;
    return arc ? history_attack<true, STAGE_SUBSET>(jobs, n_jobs, stream)
               : history_attack<false, STAGE_SUBSET>(jobs, n_jobs, stream);
}

int rcmarl_ios_pipeline_attack(const rcmarl_pipeline_attack_job* jobs, int n_jobs, int arc, void* stream) {
    if (arc != 0 && arc != 1) return RCMARL_ERR_ARG;
    return arc ? pipeline_attack<true, STAGE_IOS>(jobs, n_jobs, stream)
               : pipeline_attack<false, STAGE_IOS>(jobs, n_jobs, stream);
}

int rcmarl_ios_history_attack(const rcmarl_history_attack_job* jobs, int n_jobs, int arc, void* stream) {
    if (arc != 0 && arc != 1) return RCMARL_ERR_ARG;
    return arc ? history_attack<true, STAGE_IOS>(jobs, n_jobs, stream)
               : history_attack<false, STAGE_IOS>(jobs, n_jobs, stream);
}

int rcmarl_dissensus_attack(const rcmarl_dissensus_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    DissensusParams P;
    RangeSet S;
    int maxn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_dissensus_job& q = jobs[j];
        if (!q.dst || !q.msgs || q.n < 1 || q.n_honest < 1 || q.n_honest > RCMARL_MAX_NEIGHBOURS || q.own < 0)
            return RCMARL_ERR_ARG;
        if (bad_nodes(q.honest, q.n_honest)) return RCMARL_ERR_ARG;
        if (q.n_byz < 1 || q.n_byz > RCMARL_MAX_NEIGHBOURS || !std::isfinite(q.eps) || q.eps < 0.f) return RCMARL_ERR_ARG;
        P.jobs[j] = q;
        if (q.n > maxn) maxn = q.n;
        // writes dst, reads the own and honest rows
        S.w.floats(q.dst, q.n);
        S.r.nodes(q.msgs, &q.own, 1, q.msg_stride, q.n);
        S.r.nodes(q.msgs, q.honest, q.n_honest, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    dissensus_attack_kernel<<<dim3((maxn + 255) / 256, n_jobs), 256, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_mimic_attack(const rcmarl_mimic_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    MimicParams P;
    RangeSet S;
    int64_t max_floats = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const rcmarl_mimic_job& q = jobs[j];
        if (!q.dst || !q.msgs || !q.z || q.n < 1 || q.n_honest < 1 || q.n_honest > RCMARL_MAX_NEIGHBOURS)
            return RCMARL_ERR_ARG;
        if (bad_nodes(q.honest, q.n_honest)) return RCMARL_ERR_ARG;
        if (q.candidate_mask == 0u || (q.candidate_mask >> q.n_honest) != 0u) return RCMARL_ERR_ARG;
        if (q.update != 0 && q.update != 1) return RCMARL_ERR_ARG;
        const int64_t floats = (int64_t)(q.n_honest + 3) * q.n;
        if (floats > RCMARL_MIMIC_MAX_FLOATS) return RCMARL_ERR_ARG;
        if (floats > max_floats) max_floats = floats;
        P.jobs[j] = q;
        // writes dst, z and target_out (one int32), reads the honest rows
        S.w.floats(q.dst, q.n);
        S.w.floats(q.z, q.n);
        if (q.target_out) S.w.bytes(q.target_out, sizeof(int32_t));
        S.r.nodes(q.msgs, q.honest, q.n_honest, q.msg_stride, q.n);
    }
    if (S.overlaps()) return RCMARL_ERR_ARG;
    return launch_staged<mimic_attack_kernel>(P, n_jobs, RCMARL_MIMIC_MAX_FLOATS, max_floats, ADA_THREADS, stream);
}

int rcmarl_sgd_apply(const rcmarl_sgd_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    SgdParams P;
    int maxn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        if (!jobs[j].dst || !jobs[j].src || !jobs[j].sums || jobs[j].n < 1) return RCMARL_ERR_ARG;
        P.jobs[j] = jobs[j];
        if (jobs[j].n > maxn) maxn = jobs[j].n;
    }
    sgd_kernel<<<dim3((maxn + 255) / 256, n_jobs), 256, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_adam_apply(const rcmarl_adam_job* jobs, int n_jobs, void* stream) {
    if (!jobs || n_jobs < 1 || n_jobs > RCMARL_MAX_JOBS) return RCMARL_ERR_ARG;
    AdamParams P;
    int maxn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        if (!jobs[j].theta || !jobs[j].m || !jobs[j].v || !jobs[j].sums || jobs[j].n < 1) return RCMARL_ERR_ARG;
        P.jobs[j] = jobs[j];
        if (jobs[j].n > maxn) maxn = jobs[j].n;
    }
    adam_kernel<<<dim3((maxn + 255) / 256, n_jobs), 256, 0, (cudaStream_t)stream>>>(P);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

int rcmarl_reward_mix(const float* r, int64_t n_rows, int n_agents, const int32_t* agents, int n_listed, float scale,
                      float* out, void* stream) {
    if (!r || !out || !agents || n_rows < 0 || n_listed < 1 || n_listed > RCMARL_MAX_JOBS || n_agents < 1)
        return RCMARL_ERR_ARG;
    if (n_rows == 0) return RCMARL_OK;
    MixParams P;
    for (int k = 0; k < n_listed; ++k) {
        if (agents[k] < 0 || agents[k] >= n_agents) return RCMARL_ERR_ARG;
        P.agents[k] = agents[k];
    }
    reward_mix_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(r, n_rows, n_agents, P,
                                                                                         n_listed, scale, out);
    RC_CUDA(cudaGetLastError());
    return RCMARL_OK;
}

}  // extern "C"
