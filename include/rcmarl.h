/* rcmarl.h -- C ABI of librcmarl.so: the sm_90a kernels behind the RPBCAC
 * training hot path (reference: mfigura/Resilient-consensus-based-MARL).
 *
 * The reference has no FFI layer: its boundary is the duck-typed Python Agent
 * API (SURVEY.md 8b).  Each entry point below replaces the TensorFlow/Keras
 * library calls made by one or more reference methods (cited per function);
 * the Python mirror of the reference interface lives in
 * resilient-consensus-based-marl_b200/{agents,training,environments} and binds
 * these symbols with ctypes (INTEGRATION.md shows the stub).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless the name ends in _host;
 *  - no hidden allocation: scratch comes from the caller (`ws`, `ws_bytes`,
 *    see rcmarl_workspace_bytes); all work is stream-ordered on `stream`
 *    (a cudaStream_t passed as void*); no host synchronisation inside;
 *  - return value: 0 on success, negative rcmarl_status otherwise; nothing
 *    throws across the ABI;
 *  - all arithmetic is IEEE fp32 (FFMA on the CUDA cores; no TF32/bf16);
 *  - network parameters are packed in Keras order
 *        [W1(d_in,20) | b1(20) | W2(20,20) | b2(20) | W3(20,n_out) | b3(n_out)]
 *    with y = x @ W + b (main.py:60-82); hidden width is 20, LeakyReLU(0.1);
 *  - the replay buffer is time-major, row = t * n_envs + e (SURVEY App. C):
 *        sa [rows][3*n_agents]  = (x0,y0,a0, x1,y1,a1, ...)   train_agents.py:93
 *        ns [rows][2*n_agents]  = next state                  train_agents.py:90
 *        r  [rows][n_agents]    = scaled local rewards        train_agents.py:91
 */
#ifndef RCMARL_H
#define RCMARL_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RCMARL_HIDDEN 20
#define RCMARL_N_ACTIONS 5
#define RCMARL_MAX_JOBS 32
#define RCMARL_MAX_TERMS 3
#define RCMARL_MAX_NEIGHBOURS 16
#define RCMARL_MAX_H 7
#define RCMARL_MAX_GRID 32

typedef enum {
    RCMARL_OK = 0,
    RCMARL_ERR_ARG = -1,        /* bad argument (null pointer, size, unsupported n_agents/H) */
    RCMARL_ERR_WORKSPACE = -2,  /* workspace too small */
    RCMARL_ERR_CUDA = -3,       /* a CUDA call / launch failed: see rcmarl_last_cuda_error */
    RCMARL_ERR_NO_DEVICE = -4
} rcmarl_status;

/* which part of a buffer row feeds the network (Keras Flatten order) */
typedef enum {
    RCMARL_IN_S = 0,   /* critic / actor on s  : sa without the action column */
    RCMARL_IN_SA = 1,  /* team-reward net on sa                               */
    RCMARL_IN_NS = 2   /* critic on the next state                            */
} rcmarl_input_kind;

/* A set of buffer rows.  Contiguous: time_idx == NULL, rows = [row_begin, row_begin+n_rows).
 * Gathered mini-batch (Appendix C): row(m) = row_begin + time_idx[m / n_envs] * n_envs + m % n_envs. */
typedef struct {
    const float* sa;
    const float* ns;
    const float* r;
    int64_t row_begin;
    int64_t n_rows;
    const int32_t* time_idx;
    int32_t n_envs;
    int32_t n_agents;
} rcmarl_rows;

const char* rcmarl_version(void);
const char* rcmarl_status_string(int status);
int rcmarl_last_cuda_error(void);               /* cudaError_t of the last failure on this thread */
int rcmarl_device_info(int* sm_count, int* cc_major, int* cc_minor);
int64_t rcmarl_param_count(int d_in, int n_out); /* packed length of one network */

/* Scratch needed by the *_grad entry points for `n_jobs` jobs of at most `max_params` parameters. */
int64_t rcmarl_workspace_bytes(int n_jobs, int max_params);

/* How a one-wave grid of `sm_count` CTAs is split over `n_jobs` jobs that sweep `n_rows` buffer rows:
 * ctas_host[j] = CTAs of job j (kinds_host[j] = RCMARL_IN_*).  balanced = 0: equal shares; 1: shares sized by each
 * job's cost per row, the plan of rcmarl_grad and of rcmarl_minibatch_fit (with n_rows = one mini-batch).
 * Host arithmetic only (no device needed); exposed for tests and for sizing experiments. */
int rcmarl_grad_grid_plan(int n_agents, const int32_t* kinds_host, int n_jobs, int loss_mode, int64_t n_rows, int balanced,
                          int sm_count, int32_t* ctas_host);

/* The weight-gradient tile map of the fit kernels for a network of d_in inputs and n_out outputs ((10|15|32|48, 1) or
 * (10|32, RCMARL_N_ACTIONS)).  info[6] = {tiles, activation entries per tile, delta entries per tile, row groups per
 * warp, phase-2 warp-FFMA per 64-row chunk, first packed parameter accumulated outside the tiles (all later ones are)};
 * params[t * rows * cols + ii * cols + jj] = packed parameter index of element (ii, jj) of tile t, -1 for padding
 * (cap = capacity of params).  Host arithmetic only; exposed for tests. */
int rcmarl_grad_tile_map(int d_in, int n_out, int32_t* info, int32_t* params, int64_t cap);

/* ---------------------------------------------------------------------------
 * K4 / C5.  Coordinate-wise clipped ("winsorised") mean over the neighbour axis,
 * own value = row 0.  Replaces tf.sort/minimum/maximum/clip_by_value/reduce_mean
 * in RPBCAC_agent._resilient_aggregation (agents/resilient_CAC_agents.py:42-58).
 * vals: [n][P] with row stride `row_stride` floats; out: [P].  One streaming read.  Refused (RCMARL_ERR_ARG, nothing
 * launched, out untouched): a null vals or out, n < 1, P < 0, row_stride < P, H outside 0..RCMARL_MAX_H, H >= n.
 * P == 0 launches nothing and returns RCMARL_OK. */
int rcmarl_clip_mean(const float* vals, int n, int64_t P, int64_t row_stride, int H,
                     float* out, void* stream);

/* Resilient aggregation rule of rcmarl_consensus_hidden and rcmarl_team, applied per coordinate to the n = n_in values
 * v[0..n-1] of the in-neighbours, own = v[0].  rank(k) = #{m : v[m] < v[k] or (v[m] == v[k] and m < k)}.
 *   CLIP  the reference's clipped mean: every v[k] clipped to [min(v_(H), own), max(v_(n-H-1), own)], mean of all n
 *         (v_(r) = the value of rank r);                                                          0 <= H < n
 *   TRIM  trimmed mean: mean of the v[k] with H <= rank(k) <= n-H-1 (at H = (n-1)/2, the median);  0 <= H, 2H < n
 *   WMSR  W-MSR (LeBlanc et al., IEEE JSAC 2013): a = #{v > own}, b = #{v < own}; the v[k] with
 *         rank(k) >= n - min(H, a) or rank(k) < min(H, b) are dropped, mean of the rest.  Own and every value equal
 *         to it are kept;                                                                         0 <= H < n
 * TRIM and WMSR add the kept values in index order, so a dropped value (1e30, +-inf) never enters the result.
 * NaN inputs are not supported by any rule. */
typedef enum { RCMARL_AGG_CLIP = 0, RCMARL_AGG_TRIM = 1, RCMARL_AGG_WMSR = 2 } rcmarl_agg_rule;

/* Hidden-layer parameter consensus for many (agent, net) pairs in one launch:
 * dst[j][0:n_hidden] = aggregate (rule) over k of msgs[in_nodes[j][k]][0:n_hidden]  (own = k 0).
 * Replaces resilient_consensus_critic_hidden / _TR_hidden
 * (agents/resilient_CAC_agents.py:142-166) incl. the neighbour gather at
 * training/train_agents.py:129-130.  The output layer of dst is left untouched (:153).
 * Refused (RCMARL_ERR_ARG, nothing launched, every dst untouched): a null jobs, n_jobs outside 1..RCMARL_MAX_JOBS, a
 * null dst or msgs, n_hidden < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, H outside [0, n_in), an
 * unknown rule, TRIM with 2H >= n_in. */
typedef struct {
    float* dst;                 /* the agent's own network (packed) */
    const float* msgs;          /* base of the message stack [n_agents][msg_stride] */
    int64_t msg_stride;
    int32_t n_hidden;           /* number of leading parameters to aggregate (W1,b1,W2,b2) */
    int32_t n_in;
    int32_t H;
    int32_t in_nodes[RCMARL_MAX_NEIGHBOURS];
    int32_t rule;               /* rcmarl_agg_rule; 0 (a zero-initialised job) is CLIP */
} rcmarl_consensus_job;
int rcmarl_consensus_hidden(const rcmarl_consensus_job* jobs_host, int n_jobs, void* stream);

/* Byzantine messages crafted for one receiver (threat model: DESIGN.md section 1).  A Byzantine agent is omniscient
 * about its receiver j's neighbourhood: over the honest set S_j (the cooperative agents of in_nodes[j], in list order,
 * repeats included, n = n_honest), per packed parameter p,
 *   mu_p = (sum_k v_k,p) / n   (summed in S_j order),   sigma_p = sqrt(sum_k (v_k,p - mu_p)^2 / n)   (population std,
 * two passes), with v_k = msgs + honest[k] * msg_stride, and it sends j
 *   ALIE   (Baruch et al., NeurIPS 2019, "A Little Is Enough"), param z:   m_p = mu_p - z * sigma_p
 *   IPM    (Xie et al., UAI 2019, inner-product manipulation), param eps:  m_p = -eps * mu_p
 *   GAUSS  param s >= 0:                                                    m_p = mu_p + s * xi_p,  xi_p ~ N(0, 1)
 * xi_p comes from the rollout's counter-based Philox4x32-10 with key (seed low word, seed high word) and counter
 *   (p, attacker | receiver << 8 | 0x40000000, round, epoch)
 * (bit 30 of word 1 keeps these streams apart from the rollout's); of its output (x, y, ., .), Box-Muller takes
 * u1 = ((x >> 8) + 1) * 2^-24 in (0, 1] and u2 = (y >> 8) * 2^-24 and gives xi = sqrt(-2 ln u1) * cos(2 pi u2).  The
 * draw depends on (seed, round, epoch, attacker, receiver, p) only, never on the launch or the job order.
 * One thread per coordinate, fixed summation order, no atomics: bitwise reproducible.  dst[0:n] = m; dst must not
 * overlap the honest rows.  Refused (RCMARL_ERR_ARG, nothing launched, dst untouched): a null pointer, n < 1, n_honest
 * outside 1..RCMARL_MAX_NEIGHBOURS, a negative honest index, an unknown kind, a non-finite param, GAUSS with s < 0,
 * attacker or receiver outside 0..255 (the counter holds 8 bits of each). */
typedef enum { RCMARL_ATTACK_ALIE = 0, RCMARL_ATTACK_IPM = 1, RCMARL_ATTACK_GAUSS = 2 } rcmarl_attack_kind;
typedef struct {
    float* dst;                 /* the crafted message (packed network) */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    int32_t n;                  /* parameters crafted: dst[0:n] from msgs[honest[k]][0:n] */
    int32_t n_honest;
    int32_t honest[RCMARL_MAX_NEIGHBOURS];
    int32_t kind;               /* rcmarl_attack_kind */
    float param;                /* z, eps or s */
    uint64_t seed;              /* Philox key (GAUSS) */
    uint32_t attacker, receiver, round, epoch;   /* Philox counter words (GAUSS) */
} rcmarl_attack_job;
int rcmarl_attack(const rcmarl_attack_job* jobs_host, int n_jobs, void* stream);

/* Byzantine messages scaled to the receiver's honest spread (rcmarl_adaptive_attack): the min-max and min-sum attacks of
 * Shejwalkar & Houmansadr, "Manipulating the Byzantine" (NDSS 2021), under the threat model of rcmarl_attack.  They push
 * the message as far along a direction d as one distance constraint over the honest set allows; they do not adapt to the
 * receiver's rule or H.  All arithmetic is fp32.  Over the honest rows v_1 .. v_n (n = n_honest, in list order, repeats
 * included, v_k = msgs + honest[k] * msg_stride) with P = job.n:
 *   mu, sigma   exactly as rcmarl_attack computes them (same summation order);
 *   d           UV:  d = -mu / ||mu||, ||mu|| = sqrt(sum_p mu_p^2); d = 0 if ||mu|| is 0 or not finite
 *               STD: d = -sigma
 *               SGN: d_p = -sign(mu_p), sign(0) = 0
 *   e_k = sum_p (mu_p - v_k,p)^2,  b_k = sum_p (mu_p - v_k,p) d_p,  a = sum_p d_p^2,  D_kl = sum_p (v_k,p - v_l,p)^2;
 * each sum is taken by one warp (lane-strided fmaf partials, then the fixed xor butterfly), and a value of e_k, a, D_kl
 * or ||mu||^2 that is not finite counts as +inf.
 *   MINMAX  c = max_{k<l} D_kl (0 for n = 1); gamma_k = root(a, b_k, e_k, c); gamma = max(0, min_k gamma_k).  In exact
 *           arithmetic {g >= 0 : max_k ||mu + g d - v_k||^2 <= c} = [0, gamma] (it holds 0 because e_k <= c).
 *   MINSUM  c = max_k sum_{l != k} D_kl (summed in index order); gamma = root(n a, sum_k b_k, sum_k e_k, c) with the
 *           sums in index order and n a one fp32 product.  In exact arithmetic {g >= 0 : sum_k ||mu + g d - v_k||^2 <= c}
 *           = [0, gamma].
 * root(A, b, e, c) is the largest root of A g^2 + 2 b g + e = c in a form free of cancellation: with m = c - e and
 * R = sqrtf(fmaxf(fmaf(b, b, A * m), 0)), it is (-b + R) / A if b <= 0 and m / (b + R) otherwise; it is 0 when m <= 0.
 * gamma = 0 when a = 0, when c, a, some e_k or some b_k is not finite, or when the result is not finite.  The output is
 *   t = scale * gamma,   dst[p] = t == 0 ? mu_p : fmaf(t, d_p, mu_p),
 * so scale = 1 is the paper's attack and scale = 0 is bitwise rcmarl_attack's ALIE at z = 0.  gamma_out (optional, one
 * float) receives gamma.  The paper finds gamma by halving a step from an initial guess until the constraint holds; the
 * closed form is the supremum that search converges to.
 * One CTA per job, the honest rows, mu and d staged in shared memory, fixed summation orders, no atomics: bitwise
 * reproducible, independent of the job order and of how jobs are split over launches.  Refused (RCMARL_ERR_ARG, nothing
 * launched, dst and gamma_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a null dst or msgs, n < 1, n_honest outside
 * 1..RCMARL_MAX_NEIGHBOURS, a negative honest index, an unknown kind or dev, a scale that is not finite or is < 0,
 * (n_honest + 2) * n > RCMARL_ADAPTIVE_MAX_FLOATS (the staging bound: 16 honest rows, mu and d of up to 1536
 * parameters), a dst or gamma_out that overlaps an honest row of any job of the launch, and two written ranges (dsts,
 * gamma_outs) of the launch that overlap.  NaN inputs are not supported. */
#define RCMARL_ADAPTIVE_MAX_FLOATS (18 * 1536)
typedef enum { RCMARL_ADAPT_MINMAX = 0, RCMARL_ADAPT_MINSUM = 1 } rcmarl_adaptive_kind;
typedef enum { RCMARL_DEV_UV = 0, RCMARL_DEV_STD = 1, RCMARL_DEV_SGN = 2 } rcmarl_adaptive_dev;
typedef struct {
    float* dst;                 /* the crafted message (packed network) */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    float* gamma_out;           /* optional [1]: gamma */
    int32_t n;                  /* parameters crafted: dst[0:n] from msgs[honest[k]][0:n] */
    int32_t n_honest;
    int32_t honest[RCMARL_MAX_NEIGHBOURS];
    int32_t kind;               /* rcmarl_adaptive_kind */
    int32_t dev;                /* rcmarl_adaptive_dev */
    float scale;                /* s >= 0; 1 is the paper's attack */
    int32_t reserved;
} rcmarl_adaptive_attack_job;
int rcmarl_adaptive_attack(const rcmarl_adaptive_attack_job* jobs_host, int n_jobs, void* stream);

/* Rule-aware Byzantine messages (rcmarl_tailored_attack): the AGR-tailored attack of Shejwalkar & Houmansadr (NDSS 2021,
 * section IV; compare Fang et al., USENIX Security 2020).  Threat model: that of rcmarl_attack, extended -- the attacker
 * also knows the receiver j's aggregation rule, its H and every real message j hears.  One job is one (attacker,
 * receiver j, net).  All arithmetic is fp32.
 *   Slots.  k = 0 .. n_in-1 in in_nodes[j] order, slot 0 the receiver's own message.  slots[k] >= 0 is a real slot, the
 *           row msgs + slots[k] * msg_stride, read as it is (an honest agent, or a Malicious, Greedy or Faulty one);
 *           slots[k] = -1 is a crafted slot: a Byzantine in-neighbour of j, which the attacker models as sending the
 *           same message m as itself (repeats count).  Bit k of honest_mask marks slot k as a member of the honest set
 *           S_j; its rows, in slot order, are the honest rows of rcmarl_adaptive_attack.
 *   Search. mu, d and gamma_mm are exactly those of rcmarl_adaptive_attack for MINMAX and direction dev over S_j (the
 *           same device code and summation orders).  Gamma = scale * gamma_mm, and Gamma = 0 if that fp32 product is
 *           not finite (a huge scale: every candidate is then mu); for i = 0 .. K (K =
 *           RCMARL_TAILORED_STEPS) the candidate gamma_i = (Gamma * i) / K (fp32, in that order) and its message
 *             m(gamma_i)_p = gamma_i == 0 ? mu_p : fmaf(gamma_i, d_p, mu_p);
 *           x(gamma_i) is the slot list with every crafted slot set to m(gamma_i).
 *   Objective.  O_i = sum_p (R_j(x(gamma_i))_p - mu_p)^2, summed by one warp (lane-strided fmaf partials, then the fixed
 *           xor butterfly); a sum that is not finite counts as -inf.  R_j is the receiver's rule with H:
 *             family COORD (rule: rcmarl_agg_rule): resilient aggregation of the n_in slot values of every packed
 *               parameter, own = slot 0, as rcmarl_consensus_hidden computes it.  That is exact for the hidden layers;
 *               for the head it is the attacker's model only (the receiver combines its head through per-row
 *               estimates in rcmarl_team, which the attacker does not model);
 *             family VECTOR (rule: rcmarl_vector_rule): exactly the output of rcmarl_vector_aggregate on x(gamma_i).
 *   Output. i* = argmax_i O_i, ties to the smaller i, and i* = 0 if every O_i is -inf; dst[p] = m(gamma_i*)_p and
 *           gamma_out (optional, one float) receives gamma_i*.
 * Hence scale = 0 is bitwise rcmarl_attack's ALIE at z = 0 (mu); at scale = 1, gamma_K = gamma_mm, so the message does
 * at least as much damage to its target rule as the min-max message in the same direction (up to the rounding of O);
 * and a plain-mean receiver (COORD CLIP, H = 0) whose real slots are all honest has R_j - mu = gamma (n_crafted / n_in) d,
 * so O rises strictly with i when a = ||d||^2 > 0 and gamma_mm > 0, and the output is the min-max message at the scale.
 * (A real slot that is not honest adds a constant offset to R_j - mu, and O may fall before it rises.)
 * One CTA per job: the real slots, mu, d, the candidate and one work row staged in shared memory, fixed summation
 * orders, no atomics -- bitwise reproducible, independent of the job order and of how jobs are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst and gamma_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a null dst
 * or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, no crafted slot, no honest slot, a crafted slot marked honest,
 * a honest_mask bit at or past n_in, a slot below -1, an unknown family (RCMARL_TAILOR_SPECTRAL too: only
 * rcmarl_pipeline_attack models DnC), rule or dev, an H the rule refuses for n_in (the checks of
 * rcmarl_consensus_hidden and rcmarl_vector_aggregate), a scale that is not finite or is < 0,
 * (n_in + 3) * n > RCMARL_TAILORED_MAX_FLOATS (the staging bound: 15 real slots, mu, d, the candidate and the work row
 * of up to 1536 parameters), a dst or gamma_out that overlaps a real slot's row of any job of the launch, and two
 * written ranges (dsts, gamma_outs) of the launch that overlap.  NaN inputs are not supported. */
#define RCMARL_TAILORED_STEPS 32
#define RCMARL_TAILORED_MAX_FLOATS (19 * 1536)
typedef enum {
    RCMARL_TAILOR_COORD = 0, RCMARL_TAILOR_VECTOR = 1, RCMARL_TAILOR_SPECTRAL = 2,
    RCMARL_TAILOR_SUBSET = 3,   /* rule: rcmarl_subset_rule; only the subset forms (rcmarl_subset_pipeline_attack) */
    RCMARL_TAILOR_FILTER = 4    /* rule: rcmarl_filter_rule; only the IOS forms (rcmarl_ios_pipeline_attack) */
} rcmarl_tailored_family;
typedef struct {
    float* dst;                 /* the crafted message (packed network) */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    float* gamma_out;           /* optional [1]: gamma_i* */
    int32_t n;                  /* parameters per message */
    int32_t n_in;
    int32_t slots[RCMARL_MAX_NEIGHBOURS];   /* a message row, or -1 for a crafted slot */
    uint32_t honest_mask;       /* bit k: slot k is in the honest set */
    int32_t family;             /* rcmarl_tailored_family */
    int32_t rule;               /* rcmarl_agg_rule (COORD) or rcmarl_vector_rule (VECTOR) */
    int32_t H;
    int32_t dev;                /* rcmarl_adaptive_dev */
    float scale;                /* s >= 0: the search range is [0, s * gamma_mm] */
} rcmarl_tailored_attack_job;
int rcmarl_tailored_attack(const rcmarl_tailored_attack_job* jobs_host, int n_jobs, void* stream);

/* The dissensus attack (rcmarl_dissensus_attack) of He, Karimireddy & Jaggi, "Byzantine-robust decentralized learning
 * via ClippedGossip" (2022), under the threat model of rcmarl_attack: each Byzantine neighbour sends receiver j the
 * message that cancels (eps = 1) or reverses (eps > 1) the pull of j's honest neighbours.  One job is one (attacker,
 * receiver j, net).  All arithmetic is fp32.  With x = msgs + own * msg_stride (the receiver's own message) and the
 * honest rows v_k = msgs + honest[k] * msg_stride (S_j in list order, repeats included, S_j holding j itself), per
 * packed parameter p < n:
 *   delta_p = sum_k (v_k,p - x_p)   (summed in list order from 0),   c = eps / (float)n_byz,
 *   dst[p] = c == 0 ? x_p : fmaf(-c, delta_p, x_p),
 * so eps = 0 sends x bitwise.  n_byz is the number of entries of in_nodes[j] held by dissensus attackers (repeats
 * included): colluders split the cancellation, and under a plain mean eps = 1 leaves the receiver where it was.  This is
 * the paper's x_i - eps sum_good W_ik (x_k - x_i) / sum_byz W_ij under uniform weights.
 * One thread per coordinate, fixed summation order, no atomics: bitwise reproducible, independent of the job order and
 * of how jobs are split over launches.  Refused (RCMARL_ERR_ARG, nothing launched, dst untouched): n_jobs outside
 * 1..RCMARL_MAX_JOBS, a null dst or msgs, n < 1, n_honest outside 1..RCMARL_MAX_NEIGHBOURS, a negative honest or own
 * row, n_byz outside 1..RCMARL_MAX_NEIGHBOURS, an eps that is not finite or is < 0, a dst that overlaps an honest or own
 * row of any job of the launch, and two dsts of the launch that overlap.  NaN inputs are not supported. */
typedef struct {
    float* dst;                 /* the crafted message (packed network) */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    int32_t n;                  /* parameters crafted: dst[0:n] */
    int32_t own;                /* the receiver's message row x */
    int32_t n_honest;
    int32_t honest[RCMARL_MAX_NEIGHBOURS];
    int32_t n_byz;              /* dissensus entries of the receiver's in_nodes, repeats included */
    float eps;                  /* eps >= 0; 1 cancels the honest pull under a plain mean */
    int32_t reserved;
} rcmarl_dissensus_job;
int rcmarl_dissensus_attack(const rcmarl_dissensus_job* jobs_host, int n_jobs, void* stream);

/* The mimic attack (rcmarl_mimic_attack) of Karimireddy, He & Jaggi, "Byzantine-robust learning on heterogeneous
 * datasets via bucketing" (ICLR 2022): the attacker sends an exact copy of one honest neighbour's message, the one that
 * lies furthest along the honest messages' principal direction z, which it tracks by power iteration.  The copy is an
 * honest message, so no rule can flag it as an outlier; it over-weights one agent's view in the receiver's consensus.
 * One job is one (attacker, receiver j, net); z [n] is the job's direction state, read and written.  All arithmetic is
 * fp32; every sum over p is taken by one warp (lane-strided fmaf partials, then the fixed xor butterfly), and a sum
 * that is not finite counts as +inf.  Over the honest rows v_k = msgs + honest[k] * msg_stride (k < n_honest, in list
 * order, repeats included):
 *   Centre  mu exactly as rcmarl_attack computes it (same summation order); c_k,p = v_k,p - mu_p.
 *   Init    only when every z_p == 0: e_k = sum_p c_k,p^2, k0 = argmax_k e_k over all k (ties to the smaller k); if
 *           e_k0 is positive and finite, z_p = c_k0,p / sqrtf(e_k0), otherwise z stays 0.
 *   Step    only when update == 1 and z != 0 (after Init): one power-iteration step on the honest covariance,
 *           s_k = sum_p c_k,p z_p,  u_p = sum_k s_k c_k,p (k order, fmaf from 0),  q = sum_p u_p^2;
 *           if q is positive and finite, z_p = u_p / sqrtf(q), otherwise z is unchanged.
 *   Choose  over the candidates (bit k of candidate_mask), with the final z: t_k = sum_p c_k,p z_p, a t_k that is not
 *           finite counting as -inf; k* = argmax t_k, ties to the smaller k; k* = the lowest candidate if z = 0 or every
 *           t_k is -inf.
 *   Output  dst[0:n] = v_k* copied bitwise, z written back, target_out (optional, one int32) = k*.
 * One CTA per job: the centred honest rows, mu, z and u staged in shared memory, fixed summation orders, no atomics:
 * bitwise reproducible, independent of the job order and of how jobs are split over launches.  Jobs with equal inputs
 * (colluding attackers of one receiver) keep bitwise equal states and copy the same row.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst, z and target_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a
 * null dst, msgs or z, n < 1, n_honest outside 1..RCMARL_MAX_NEIGHBOURS, a negative honest row, an empty candidate_mask
 * or one with a bit at or past n_honest, update other than 0 or 1, (n_honest + 3) * n > RCMARL_MIMIC_MAX_FLOATS (the
 * staging bound: 16 honest rows, mu, z and u of up to 1536 parameters), a dst, z or target_out that overlaps an honest
 * row of any job of the launch, and two written ranges (dsts, zs, target_outs) of the launch that overlap.  NaN inputs
 * are not supported. */
#define RCMARL_MIMIC_MAX_FLOATS (19 * 1536)
typedef struct {
    float* dst;                 /* the copied message (packed network) */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    float* z;                   /* [n] direction state, read and written; all zero: not yet initialised */
    int32_t* target_out;        /* optional [1]: k* */
    int32_t n;                  /* parameters per message */
    int32_t n_honest;
    int32_t honest[RCMARL_MAX_NEIGHBOURS];
    uint32_t candidate_mask;    /* bit k: honest entry k may be copied */
    int32_t update;             /* 1: take one power step; 0: keep z (after Init) */
} rcmarl_mimic_job;
int rcmarl_mimic_attack(const rcmarl_mimic_job* jobs_host, int n_jobs, void* stream);

/* Distance-based resilient aggregation of whole messages (rcmarl_vector_aggregate).  The rules above are coordinate-wise;
 * these compare the in-neighbours' messages as vectors.  One job: its n = n_in messages x_k = msgs + in_nodes[k] *
 * msg_stride, k = 0 .. n-1 (k = 0 is the receiver's own; repeats in in_nodes count), each of P = job.n packed
 * parameters (the whole network, hidden layers and head).  In fp32:
 *   D_kl = sum_p (x_k,p - x_l,p)^2,   d_k(z) = sqrt(sum_p (x_k,p - z_p)^2);
 * a distance that is not finite (overflow, e.g. a message of 1e30, or +-inf) counts as +inf, and a term (x_k,p -
 * x_l,p)^2 below the fp32 range rounds to 0 (messages that differ by less than about 1e-23 per coordinate are at
 * distance 0, and the index tie rules decide).  Every rule outputs
 *   out = sum_k w_k x_k,   w_k >= 0,   sum_k w_k = 1,
 * and writes w to weights_out when it is not NULL.
 *   KRUM    (Blanchard et al., NeurIPS 2017)  n >= H + 3.  score_k = the sum of the n - H - 2 smallest D_kl over l != k,
 *   MKRUM   added in ascending order.  The m smallest scores are selected (ties to the lower index), m = 1 for KRUM and
 *           m = n - H for MKRUM (multi-Krum); out = (sum over the selected k, index order, of x_k) / m, w_k = 1/m or 0.
 *   SCCLIP  self-centred clipping (after He, Karimireddy & Jaggi 2022, ClippedGossip).  The clipping radius is set by H,
 *           not by the paper's adaptive rule (this library's choice): d_k = d_k(x_0) for k >= 1, tau = the (H+1)-th
 *           largest d_k (0 if H >= n - 1), c_k = 0 if d_k is not finite, 1 if d_k <= tau, tau / d_k otherwise;
 *           out = x_0 + (sum_{k>=1, index order, c_k != 0} c_k (x_k - x_0)) / n, w_k = c_k / n (k >= 1),
 *           w_0 = 1 - sum_{k>=1} w_k.  H = 0 gives the plain mean.
 *   GMED    geometric median by smoothed Weiszfeld (Pillutla et al., RFA).  z^0 = the coordinate-wise median (TRIM at
 *           H' = (n-1)/2); then RCMARL_GMED_ITERS times: beta_k = 0 if d_k(z) is not finite, else
 *           1 / max(d_k(z), RCMARL_GMED_NU), z <- (sum_k beta_k x_k) / sum_k beta_k (index order, beta_k = 0 terms
 *           skipped); out = the last z, w_k = the last beta_k / sum beta.  If no distance is finite, beta = (1, 0, ...):
 *           out = x_0.  H is not used (0 <= H < n).
 * NaN inputs are not supported.  At most H messages of 1e30 or +-inf get weight 0 (KRUM / MKRUM: while n >= 2H + 3;
 * GMED: while 2H < n).  One CTA per job, fixed summation orders, no atomics: bitwise reproducible, independent of the
 * job order and of how jobs are split over launches.  dst[0:n] = out.  Refused (RCMARL_ERR_ARG, nothing launched, dst
 * and weights_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a null dst or msgs, n < 1, n_in outside
 * 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, an unknown rule, H outside [0, n_in), KRUM / MKRUM with n_in < H + 3,
 * (n_in + 1) * n > RCMARL_VECTOR_MAX_FLOATS (the messages are staged in shared memory), a dst or weights_out that
 * overlaps an in-node row of any job of the launch, and two written ranges (dsts, weights_outs) of the launch that
 * overlap. */
#define RCMARL_GMED_ITERS 8
#define RCMARL_GMED_NU 1e-6f
#define RCMARL_VECTOR_MAX_FLOATS (48 * 1024)
typedef enum { RCMARL_VEC_KRUM = 0, RCMARL_VEC_MKRUM = 1, RCMARL_VEC_SCCLIP = 2, RCMARL_VEC_GMED = 3 } rcmarl_vector_rule;
typedef struct {
    float* dst;                 /* the aggregate (packed network) */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    float* weights_out;         /* optional [n_in]: w_k */
    int32_t n;                  /* parameters per message */
    int32_t n_in;
    int32_t H;
    int32_t rule;               /* rcmarl_vector_rule */
    int32_t in_nodes[RCMARL_MAX_NEIGHBOURS];
} rcmarl_vector_job;
int rcmarl_vector_aggregate(const rcmarl_vector_job* jobs_host, int n_jobs, void* stream);

/* Spectral resilient aggregation of whole messages (rcmarl_dnc_aggregate): the divide-and-conquer (DnC) rule of
 * Shejwalkar & Houmansadr, "Manipulating the Byzantine" (NDSS 2021, section VI, Algorithm 2), which removes the messages
 * that lie furthest along the top principal direction of the centred messages.  It takes rcmarl_vector_job with
 * rule = RCMARL_SPECTRAL_DNC; its n = n_in messages x_0 .. x_{n-1} (x_0 the receiver's own; repeats in in_nodes count)
 * each hold P = job.n packed parameters.
 *   Flagged  F = the rows holding +-inf; U = every other row, in index order, m = |U|.  If m = 0: out = x_0, w = e_0.
 *   Centre   in fp64 from the fp32 inputs: mu_p = (sum_{k in U, index order} x_k,p) / m,  c_k = x_k - mu (k in U),
 *            G_kl = sum_p c_k,p c_l,p (each G_kl summed by one warp: lane-strided fma partials, then the fixed xor
 *            butterfly).  fp64 holds the square of any finite fp32 value, so only +-inf needs flagging.
 *   Scores   lambda = the largest eigenvalue of G and u its unit eigenvector, by cyclic Jacobi in fp64 (rows p < q
 *            in order; a rotation is skipped, and G_pq set to 0, when 100 |G_pq| is below the rounding of |G_pp| and
 *            of |G_qq|; at most RCMARL_DNC_SWEEPS sweeps, ending early after a sweep without a rotation); lambda is
 *            the largest diagonal entry (ties to the lower index).  score_k = lambda u_k^2 = <c_k, v>^2 for k in U (v
 *            the top right singular vector of the centred rows, the paper's outlier score); score_k = +inf for k in F.
 *   Removal  max(|F|, H) rows are removed: every row of F, then the H - |F| highest scores of U (equal scores: the
 *            higher index first).  I = the kept rows.
 *   Output   out = (sum_{k in I, index order} x_k) / |I| in fp32 (as multi-Krum's), w_k = 1/|I| on I, 0 elsewhere;
 *            weights_out receives w when it is not NULL.
 * 0 <= H < n_in; H = 0 gives the plain mean, and the rule may remove the receiver's own message.  Every coordinate is
 * used in one iteration that removes H rows (the paper's b = P, niters = 1 and c = 1, with H as its bound m on the
 * number of malicious messages): with every coordinate, each further iteration would pick the same rows.  When lambda is repeated or nearly so, u (and
 * so the selection) is not unique: which of the candidate directions the Jacobi sweep returns is fixed, but it is not
 * a property of the messages.  NaN inputs are not supported.  One CTA per job, fixed summation orders, no atomics:
 * bitwise reproducible, independent of the job order and of how jobs are split over launches.  dst[0:n] = out.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst and weights_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a null
 * dst or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, a rule other than RCMARL_SPECTRAL_DNC,
 * H outside [0, n_in), (n_in + 2) * n > RCMARL_DNC_MAX_FLOATS (the staging bound: the fp32 messages and the fp64 mean
 * are staged in shared memory), a dst or weights_out that overlaps an in-node row of any job of the launch, and two
 * written ranges (dsts, weights_outs) of the launch that overlap. */
#define RCMARL_DNC_SWEEPS 32
#define RCMARL_DNC_MAX_FLOATS (48 * 1024)
typedef enum { RCMARL_SPECTRAL_DNC = 0 } rcmarl_spectral_rule;
int rcmarl_dnc_aggregate(const rcmarl_vector_job* jobs_host, int n_jobs, void* stream);

/* Exact subset-selection aggregation of whole messages (rcmarl_subset_aggregate): average the n - H messages that agree
 * most as a set, found by searching every subset.  MDA, minimum-diameter averaging (El-Mhamdi, Guerraoui & Rouault,
 * ICLR 2021), picks the subset of smallest diameter; SMEA, smallest-maximum-eigenvalue averaging (Allouah, Guerraoui,
 * Gupta, Pinot & Stephan, ICML 2023), the subset whose covariance has the smallest top eigenvalue.  It takes
 * rcmarl_vector_job with rule = RCMARL_SUBSET_MDA or RCMARL_SUBSET_SMEA; its n = n_in messages x_0 .. x_{n-1}, x_k =
 * msgs + in_nodes[k] * msg_stride (x_0 the receiver's own; repeats in in_nodes count) each hold P = job.n floats.
 *   Flagged    F = the rows holding +-inf (DnC's convention); U = every other row, in index order.  If U is empty:
 *              out = x_0, w = e_0.  A row of 1e30 is finite and not flagged: fp64 holds its squared distances.
 *   Distances  D_kl = sum_p ((double)x_k,p - (double)x_l,p)^2 for k, l in U, in fp64 (each pair summed by one warp:
 *              lane-strided fma partials, then the fixed xor butterfly).  D_kk = 0, not computed.
 *   Candidates s = n - max(|F|, H) (>= 1, as 0 <= H < n); the candidates are every s-subset of U, ranked in the
 *              lexicographic order of their sorted index lists.
 *   Criterion  c(S) = 0 when s = 1.  Otherwise MDA: c(S) = max over a < b in S of D_ab.  SMEA: c(S) = lambda_max(B_S),
 *              B_S = -1/2 J D_S J the double-centred squared-distance matrix, in fp64 in this order: r_a = (sum_{b in
 *              S, in order} D_ab) / s, t = (sum_{a in S, in order} r_a) / s, B_ab = -0.5 * (((D_ab - r_a) - r_b) + t)
 *              for positions a <= b in S, B_ba = B_ab; lambda_max by cyclic Jacobi with exactly DnC's rotation and skip
 *              rules and at most RCMARL_DNC_SWEEPS sweeps, the largest diagonal entry.  The covariance's top
 *              eigenvalue is lambda_max / s; every candidate has the same s, so the 1/s is dropped.
 *   Selection  S* = argmin c(S), ties to the lower rank.
 *   Output     out = (sum_{k in S*, index order} x_k) / (float)s, an fp32 sum from 0 (multi-Krum's and DnC's
 *              arithmetic); w_k = 1/(float)s on S*, 0 elsewhere, written to weights_out when it is not NULL.
 * H = 0 with no flagged row gives the plain mean, bitwise rcmarl_dnc_aggregate's at H = 0 and, where n_in >= 3,
 * multi-Krum's at H = 0.  H = n - 1 with no flagged row gives x_0 bitwise (a -0 coordinate comes out +0, as the sum
 * starts from 0): every criterion is 0 and rank 0 is {0}.  The rule may drop the receiver's own message.  Rows of +-inf
 * are never selected while fewer than n_in rows hold them, and rows of 1e30, at most H of them, get weight 0 while the
 * other rows lie far closer together (a 1e30 row is at a squared distance of about 1e60 from each of them).  NaN inputs
 * are not supported.  At most C(16, 8) = 12 870 candidates per job; one CTA per job, fixed summation orders, no
 * atomics: bitwise reproducible, independent of the job order and of how jobs are split over launches.  dst[0:n] = out.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst and weights_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a null
 * dst or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, a rule other than RCMARL_SUBSET_MDA and
 * RCMARL_SUBSET_SMEA, H outside [0, n_in), n_in * n > RCMARL_SUBSET_MAX_FLOATS (the staging bound: the messages are
 * staged in shared memory), a dst or weights_out that overlaps an in-node row of any job of the launch, and two written
 * ranges (dsts, weights_outs) of the launch that overlap. */
#define RCMARL_SUBSET_MAX_FLOATS (48 * 1024)
typedef enum { RCMARL_SUBSET_MDA = 0, RCMARL_SUBSET_SMEA = 1 } rcmarl_subset_rule;
int rcmarl_subset_aggregate(const rcmarl_vector_job* jobs_host, int n_jobs, void* stream);

/* Iterative outlier scissor (rcmarl_ios_aggregate): the IOS rule of Wu, Chen & Ling, "Byzantine-Resilient
 * Decentralized Stochastic Optimization With Robust Aggregation Rules" (IEEE Trans. Signal Processing, 2023), with
 * uniform weights (so FABA, Xia et al., IJCAI 2019, over one neighbourhood).  The receiver drops the message furthest
 * from the mean of those it still holds, re-centres, and repeats H times; the output is the mean of the rest.  It takes
 * rcmarl_vector_job with rule = RCMARL_FILTER_IOS; its n = n_in slots x_0 .. x_{n-1}, x_k = msgs + in_nodes[k] *
 * msg_stride (x_0 the receiver's own; repeats in in_nodes count) each hold P = job.n floats.
 *   Flagged  F = the rows holding +-inf (DnC's convention); U = every other row, in index order.  If U is empty:
 *            out = x_0, w = e_0.  A row of 1e30 is finite and not flagged: fp64 holds the square of any finite fp32
 *            value, so it is removed by its distance.
 *   Iterate  max(0, H - |F|) times: the centre c_p = (sum_{k in U, index order} (double)x_k,p) / (double)|U| in fp64,
 *            from scratch; d_k = sum_p ((double)x_k,p - c_p)^2 for k in U (each d_k summed by one warp: lane-strided
 *            fma partials, then the fixed xor butterfly); remove k* = argmax_{k in U} d_k (equal d: the higher index
 *            first) from U.
 *   Output   I = the rows left in U; out = (sum_{k in I, index order} x_k) / (float)|I|, an fp32 sum from 0
 *            (multi-Krum's, DnC's and MDA's arithmetic); w_k = 1/(float)|I| on I, 0 elsewhere, written to weights_out
 *            when it is not NULL.
 * The receiver's own message is a candidate for removal, as under DnC and MDA: this is the library's definition.  It
 * differs from the paper's Algorithm 1, where the receiver removes only received messages and always keeps its own.  Two rows
 * left lie equally far from their mean: where their fp64 sums are exact (coordinate exponents less than 29 apart), the
 * two d are equal and the higher index is removed.  H = 0
 * with no flagged row gives the plain mean, bitwise rcmarl_dnc_aggregate's and rcmarl_subset_aggregate's at H = 0 and,
 * where n_in >= 3, multi-Krum's at H = 0.  Rows of +-inf are never kept while fewer than n_in rows hold them, and rows
 * of 1e30, at most H - |F| of them, get weight 0 while the other rows lie far closer together.  NaN inputs are not
 * supported.  One CTA per job, fixed summation orders, no atomics: bitwise reproducible, independent of the job order
 * and of how jobs are split over launches.  dst[0:n] = out.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst and weights_out untouched): n_jobs outside 1..RCMARL_MAX_JOBS, a null
 * dst or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, a rule other than RCMARL_FILTER_IOS,
 * H outside [0, n_in), (n_in + 2) * n > RCMARL_IOS_MAX_FLOATS (the staging bound: the fp32 messages and the fp64 centre
 * are staged in shared memory), a dst or weights_out that overlaps an in-node row of any job of the launch, and two
 * written ranges (dsts, weights_outs) of the launch that overlap. */
#define RCMARL_IOS_MAX_FLOATS (48 * 1024)
typedef enum { RCMARL_FILTER_IOS = 0 } rcmarl_filter_rule;
int rcmarl_ios_aggregate(const rcmarl_vector_job* jobs_host, int n_jobs, void* stream);

/* Nearest-neighbour mixing (rcmarl_nnm_mix): the pre-aggregation step of Allouah, Farhadkhani, Guerraoui, Gupta, Pinot
 * & Stephan, "Fixing by Mixing: A Recipe for Optimal Byzantine ML under Heterogeneity" (AISTATS 2023).  It replaces each
 * message a receiver hears by the mean of its n - H nearest received messages (itself among them); the receiver's own
 * rule then runs on the mixed messages.  It takes rcmarl_vector_job with rule = RCMARL_MIX_NNM; its n = n_in messages
 * x_0 .. x_{n-1} (x_0 the receiver's own; repeats in in_nodes count) each hold P = job.n packed parameters.  In fp32:
 *   D_kl     for k != l exactly as rcmarl_vector_aggregate computes it (each pair k < l summed by one warp, lane-strided
 *            partials, then the fixed xor butterfly); a distance that is not finite counts as +inf.  D_kk = 0, not
 *            computed (a row holding +-inf gives no NaN).
 *   N_k      order l by (D_kl, then l != k, then l) -- the own row first among equal distances, then the lower index --
 *            and take the first n - H, less every l with D_kl = +inf.  N_k always holds k.
 *   Output   mixed_k = (sum_{l in N_k, index order} x_l) / |N_k|: an fp32 sum from 0, then one division by
 *            (float)|N_k| (multi-Krum's arithmetic), written to dst + k * msg_stride for k = 0 .. n-1.  weights_out,
 *            when not NULL, receives M row-major [n_in][n_in]: M_kl = 1/|N_k| for l in N_k, 0 elsewhere.
 * 0 <= H < n_in.  H = 0 with every distance finite gives every row multi-Krum's output at H = 0 (the plain mean); H =
 * n - 1 passes every row through.  A row at non-finite distance from every other row (+-inf, 1e30) passes through and
 * no finite row mixes it in, so at most H poisoned inputs give at most H poisoned mixed rows.  NaN inputs are not
 * supported.  One CTA per job, fixed summation orders, no atomics: bitwise reproducible, independent of the job order
 * and of how jobs are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, every dst row and weights_out untouched): n_jobs outside
 * 1..RCMARL_MAX_JOBS, a null dst or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, a rule
 * other than RCMARL_MIX_NNM, H outside [0, n_in), n_in * n > RCMARL_NNM_MAX_FLOATS (the messages are staged in shared
 * memory), a written range (the n_in dst rows, the n_in^2 weights) that overlaps an in-node row of any job of the
 * launch, and two written ranges of the launch that overlap. */
#define RCMARL_NNM_MAX_FLOATS (48 * 1024)
typedef enum { RCMARL_MIX_NNM = 0, RCMARL_MIX_BUCKET = 1, RCMARL_MIX_MOMENTUM = 2, RCMARL_MIX_ARC = 3 } rcmarl_mixing_rule;
int rcmarl_nnm_mix(const rcmarl_vector_job* jobs_host, int n_jobs, void* stream);

/* Adaptive robust clipping (rcmarl_arc_clip): the pre-aggregation step of Allouah et al., "Boosting Robustness by
 * Clipping Gradients in Distributed Learning" (2024).  Before the receiver's rule runs,
 * the k_clip received messages furthest from its own are pulled in along the line to its own message, to the distance
 * of the (k_clip + 1)-th furthest; k_clip follows from H alone.  The paper clips gradient norms around the origin; the
 * messages here are parameters, so ARC clips each message's offset from the receiver's own row.  It takes
 * rcmarl_vector_job with rule = RCMARL_MIX_ARC; one job is one (receiver, net): n = n_in slots x_k = msgs + in_nodes[k]
 * * msg_stride (x_0 the receiver's own; repeats in in_nodes count as separate slots), each of P = job.n floats,
 * 0 <= H < n_in.  In fp32:
 *   d_k      = sqrtf(squared distance of x_k and x_0) for k >= 1, the squared distance summed exactly as
 *            rcmarl_vector_aggregate sums scclip's (one warp, lane-strided partials, then the fixed xor butterfly), so
 *            d_k is bitwise scclip's d_k; a d_k that is not finite counts as +inf.
 *   k_clip   = (2 * H * (n - H)) / n in integer division: the paper's floor(2 (f/n) (n - f)) at f = H (n = 4, H = 1: 1).
 *   tau      = the (k_clip + 1)-th largest of d_1 .. d_{n-1}, or 0 if k_clip >= n - 1.
 *   c_k      c_0 = 1; c_k = 0 if d_k is not finite, 1 if d_k <= tau, else tau / d_k (one IEEE division, __fdiv_rn).
 *   Output   row k at dst + k * msg_stride: x_k bitwise if c_k = 1 (row 0 always), x_0 bitwise if c_k = 0, else
 *            x_0,p + c_k * (x_k,p - x_0,p) with every operation rounded on its own (no FMA).  weights_out, when not
 *            NULL, receives c [n_in].
 * H = 0 passes every row through bitwise.  At most k_clip finite rows change, and a changed row lies at distance tau
 * from x_0 up to rounding.  A +-inf or 1e30 message becomes x_0, so poisoned inputs never give poisoned rows.  NaN
 * inputs are not supported.  Nothing is staged in shared memory, so P has no bound of its own.  One CTA per job, fixed
 * summation orders, no atomics: bitwise reproducible, independent of the job order and of how jobs are split over
 * launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, every dst row and weights_out untouched): n_jobs outside
 * 1..RCMARL_MAX_JOBS, a null dst or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, a rule
 * other than RCMARL_MIX_ARC, H outside [0, n_in), a written range (the n_in dst rows, the n_in weights) that overlaps an
 * in-node row of any job of the launch, and two written ranges of the launch that overlap. */
int rcmarl_arc_clip(const rcmarl_vector_job* jobs_host, int n_jobs, void* stream);

/* Randomized bucketing (rcmarl_bucket_mix): the pre-aggregation step of Karimireddy, He & Jaggi, "Byzantine-robust
 * learning on heterogeneous datasets via bucketing" (ICLR 2022).  The messages a receiver hears are shuffled into
 * buckets of s and each bucket is replaced by its mean; the receiver's own rule then runs on the bucket means.  Unlike
 * the paper, the receiver's own message x_0 -- the one row it knows to be honest -- passes through and is not bucketed,
 * so n_in = 4 at s = 2 gives the rule 3 rows.  One job is one (receiver, net): n = n_in message slots x_0 .. x_{n-1},
 * x_k = msgs + in_nodes[k] * msg_stride (x_0 the receiver's own; repeats in in_nodes count), each of P = job.n packed
 * parameters.  All arithmetic is fp32.  With m = n - 1:
 *   Permutation  pi = [1, .., m] shuffled by Fisher-Yates for i = m-1 down to 1 (0-based positions): draw t (t = 0 for
 *            the first swap) is the 32-bit word u = word (t & 3) of Philox4x32-10 with key (seed low word, seed high
 *            word) and counter (t >> 2, receiver | net << 8 | 0x20000000, round, epoch); j = (u * (i + 1)) >> 32 in 64
 *            bits, and pi[i], pi[j] are swapped.  Bit 29 of word 1 keeps the stream apart from the rollout's and from
 *            rcmarl_attack's (bit 30).  The draw depends on (seed, round, epoch, receiver, net) only, never on the
 *            launch or the job order.
 *   Buckets  B = ceil(m / s); bucket b holds the slots pi[b*s .. min((b+1)*s, m) - 1].
 *   Output   n_out = 1 + B rows at dst + r * msg_stride: row 0 = x_0 bitwise; row 1 + b = (sum of bucket b's members,
 *            in increasing slot order (not pi order), an fp32 sum from 0) / (float)|bucket b| (multi-Krum's and
 *            rcmarl_nnm_mix's arithmetic; the paper's 1/s when s divides m).  If any coordinate of that mean is not
 *            finite, every coordinate of row 1 + b is +inf, so at most H poisoned inputs give at most H poisoned rows.
 *            weights_out, when not NULL, receives M row-major [n_out][n_in]: M_00 = 1, M_(1+b)l = 1/|bucket b| for
 *            every slot l in bucket b, 0 elsewhere.
 * n_in = 1 gives the own row only; s >= m a single bucket (the mean of every received message); s = 1 the received
 * messages in permuted order, each copied bitwise.  NaN inputs are not supported.  One CTA per job, the permutation in
 * shared memory, fixed summation orders, no atomics: bitwise reproducible, independent of the job order and of how jobs
 * are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, every dst row and weights_out untouched): n_jobs outside
 * 1..RCMARL_MAX_JOBS, a null dst or msgs, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, s < 1, net
 * other than 0 or 1, receiver > 255, a written range (the n_out dst rows, the n_out * n_in weights) that overlaps an
 * in-node row of any job of the launch, and two written ranges of the launch that overlap. */
typedef struct {
    float* dst;                 /* n_out rows at dst + r * msg_stride */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    float* weights_out;         /* optional [n_out * n_in]: M */
    int32_t n;                  /* parameters per message */
    int32_t n_in;
    int32_t s;                  /* bucket size, >= 1 */
    int32_t in_nodes[RCMARL_MAX_NEIGHBOURS];
    uint64_t seed;              /* Philox key */
    uint32_t receiver, net, round, epoch;   /* Philox counter words */
} rcmarl_bucket_job;
int rcmarl_bucket_mix(const rcmarl_bucket_job* jobs_host, int n_jobs, void* stream);

/* Per-neighbour momentum (rcmarl_momentum_mix): the stateful pre-aggregation step of Karimireddy, He & Jaggi, "Learning
 * from History for Byzantine Robust Optimization" (ICML 2021).  The receiver keeps, for every slot it hears, an
 * exponential moving average of that slot's update against its own net, and its rule reads the averages instead of the
 * latest messages: honest noise averages out, a bias repeated every round builds up into an outlier.  Momentum is
 * linear in what the receiver hears, so the receiver computes it itself; what agents send is unchanged.  One job is one
 * (receiver, net): n = n_in message slots x_k = msgs + in_nodes[k] * msg_stride (x_0 the receiver's own; repeats in
 * in_nodes count as separate slots), each of P = job.n floats; the reference c = ref[0:P] (the receiver's net after its
 * previous consensus step); the state M, n_in rows at momentum + k * momentum_stride, read and written; beta in [0, 1)
 * and first in {0, 1}.  For each slot k and coordinate p, in fp32 with every operation rounded on its own (no FMA):
 *   u       = x_k,p - c_p
 *   M_k,p   = u                             if first, or if M_k,p is finite and u is not
 *           = M_k,p                         if M_k,p is +-inf and not first (a poisoned coordinate stays poisoned)
 *           = beta * M_k,p + (1 - beta) * u otherwise ((1 - beta) one fp32 subtraction)
 *   row_k,p = c_p + M_k,p                   written to dst + k * msg_stride.
 * The rows are full packed nets (row 0 the own slot's), read by every rule as the mixed rows of rcmarl_nnm_mix are.  A
 * +-inf or 1e30 message poisons its own slot's row only, so at most H poisoned inputs give at most H poisoned rows.  At
 * beta = 0, row_k = (x_k - c) + c: x_k up to one rounding.  first = 1 ignores the old M (it is not read).  NaN inputs
 * are not supported.  One thread per coordinate and slot, no reductions, no atomics: bitwise reproducible, independent
 * of the job order and of how jobs are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, every dst row and every M row untouched): n_jobs outside
 * 1..RCMARL_MAX_JOBS, a null dst, msgs, ref or momentum, n < 1, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative
 * in-node, a beta that is not finite or lies outside [0, 1), first other than 0 or 1, a written range (the n_in dst
 * rows, the n_in M rows) that overlaps an in-node row or a ref of any job of the launch, two written ranges of the
 * launch that overlap, and a ref that overlaps an in-node row of any job of the launch. */
typedef struct {
    float* dst;                 /* n_in rows at dst + k * msg_stride */
    const float* msgs;          /* base of the message stack */
    int64_t msg_stride;
    const float* ref;           /* [n]: c */
    float* momentum;            /* n_in rows at momentum + k * momentum_stride: M, read and written */
    int64_t momentum_stride;
    int32_t n;                  /* parameters per message */
    int32_t n_in;
    int32_t in_nodes[RCMARL_MAX_NEIGHBOURS];
    float beta;                 /* 0 <= beta < 1 */
    int32_t first;              /* 1: M = u (the slot's first step) */
} rcmarl_momentum_job;
int rcmarl_momentum_mix(const rcmarl_momentum_job* jobs_host, int n_jobs, void* stream);

/* Pipeline-aware Byzantine messages (rcmarl_pipeline_attack): the AGR-tailored attack of rcmarl_tailored_attack against
 * the receiver's whole aggregation pipeline -- its mixing step (none, rcmarl_nnm_mix or rcmarl_bucket_mix), then its rule,
 * DnC included.  Threat model: that of rcmarl_tailored_attack, plus the receiver's mixing step; a bucketing receiver's
 * shuffle stays secret (it is that defence's premise), so the attacker draws shuffles of its own.  One job is one
 * (attacker, receiver j, net); `attack` holds the fields of rcmarl_tailored_attack_job with their meaning there.  All
 * arithmetic is fp32 (DnC's centring and eigen-solve fp64, as in rcmarl_dnc_aggregate).
 *   Search.  mu, d, gamma_mm, Gamma, the K + 1 candidates gamma_i, m(gamma_i) and the slot list x(gamma_i) exactly as in
 *           rcmarl_tailored_attack (the same device code and summation orders).
 *   Mixing.  x(gamma_i) is mixed first, and the rule then reads the mixed rows with H:
 *             RCMARL_PIPE_NONE    the n_in slots (n_rows = n_in);
 *             RCMARL_PIPE_NNM     the n_in mixed rows of rcmarl_nnm_mix at H, bitwise (n_rows = n_in);
 *             RCMARL_PIPE_BUCKET  the own slot, then the bucket means exactly as rcmarl_bucket_mix computes them (the
 *                                 +inf poisoned rows included) under the attacker's sample q of the shuffle
 *                                 (n_rows = 1 + ceil((n_in - 1) / s)).
 *           Sample q < n_perms is the Fisher-Yates of rcmarl_bucket_mix whose draw t is word t & 3 of Philox4x32-10 with
 *           key (seed low word, seed high word) and counter ((q << 2) | (t >> 2), attacker | receiver << 8 | net << 16 |
 *           0x10000000, round, epoch).  Bit 28 of word 1 keeps this stream apart from rcmarl_bucket_mix's (bit 29),
 *           rcmarl_attack's (bit 30) and the rollout's resets (bit 31).  Without bucketing there is one sample.
 *   Rule.    family COORD: resilient_mean per coordinate over the n_rows rows (rcmarl_consensus_hidden's arithmetic);
 *           VECTOR: exactly rcmarl_vector_aggregate's output; SPECTRAL (rule RCMARL_SPECTRAL_DNC): exactly
 *           rcmarl_dnc_aggregate's output.  R_q(gamma_i) is the rule's output on sample q.
 *   Objective.  O_i,q = sum_p (R_q(gamma_i)_p - mu_p)^2 as in rcmarl_tailored_attack (-inf if not finite);
 *           Obar_i = (sum_q O_i,q, q order, an fp32 sum from 0) / (float)n_perms, -inf if some O_i,q is -inf or Obar_i
 *           is not finite.  i* = argmax_i Obar_i, ties to the smaller i, i* = 0 if every Obar_i is -inf.
 *   Output.  dst[0:n] = m(gamma_i*), gamma_out (optional, one float) = gamma_i*, model_out (optional, n floats) =
 *           R_0(gamma_i*): the receiver's aggregate as the attacker models it (under bucketing, with sample 0).
 * With mixing none and family COORD or VECTOR, dst and gamma_out are bitwise those of rcmarl_tailored_attack.  A
 * zero-initialised mixing field is RCMARL_PIPE_NONE; s, n_perms and the Philox words are read only under bucketing.
 * One CTA per job: the real slots, mu, d, the candidate, the output row, the mixed rows and (DnC) the fp64 mean staged
 * in shared memory, fixed summation orders, no atomics -- bitwise reproducible, independent of the job order and of how
 * jobs are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst, gamma_out and model_out untouched): everything rcmarl_tailored_attack
 * refuses (family SPECTRAL with rule RCMARL_SPECTRAL_DNC excepted; its H must lie in [0, n_rows)), an unknown mixing,
 * an H the rule refuses at n_rows, under bucketing s < 1, n_perms outside 1..RCMARL_PIPELINE_MAX_PERMS, attacker or
 * receiver > 255 or net other than 0 or 1, a staging size (n_real + n_mixed + 4 + (DnC ? 2 : 0)) * n above
 * RCMARL_PIPELINE_MAX_FLOATS (n_real the real slots; n_mixed = 0 without mixing, n_in under nnm and n_rows - 1 under
 * bucketing, whose own row is read in place; the bound admits the 16-agent team-reward net, 1421 parameters, at n_in =
 * 16 under nnm with any family), a written range (dst, gamma_out, model_out) that overlaps a real slot's row of any job
 * of the launch, and two written ranges of the launch that overlap.  NaN inputs are not supported. */
#define RCMARL_PIPELINE_MAX_FLOATS (37 * 1421)
#define RCMARL_PIPELINE_MAX_PERMS 16
typedef enum { RCMARL_PIPE_NONE = 0, RCMARL_PIPE_NNM = 1, RCMARL_PIPE_BUCKET = 2 } rcmarl_pipeline_mixing;
typedef struct {
    rcmarl_tailored_attack_job attack;   /* family COORD, VECTOR or SPECTRAL; slots, H and dev as for the tailored attack */
    float* model_out;           /* optional [n]: R_0(gamma_i*) */
    uint64_t seed;              /* Philox key (bucketing) */
    int32_t mixing;             /* rcmarl_pipeline_mixing; 0 (a zero-initialised job) is none */
    int32_t s;                  /* bucket size, >= 1 (bucketing) */
    int32_t n_perms;            /* the attacker's shuffle samples, 1..RCMARL_PIPELINE_MAX_PERMS (bucketing) */
    uint32_t attacker, receiver, net, round, epoch;   /* Philox counter words (bucketing) */
} rcmarl_pipeline_attack_job;
int rcmarl_pipeline_attack(const rcmarl_pipeline_attack_job* jobs_host, int n_jobs, void* stream);

/* Momentum-aware Byzantine messages (rcmarl_history_attack): the pipeline attack without mixing, run in the momentum-row
 * space of a receiver j with per-neighbour momentum (rcmarl_momentum_mix), then inverted through j's momentum step.
 * Threat model: that of rcmarl_pipeline_attack, plus j's momentum: the attacker knows beta, j's reference net c, its
 * state M and whether this is its first step -- functions of messages an omniscient attacker has already seen.  The
 * attack is greedy per epoch; it does not plan across epochs.  One job is one (attacker, receiver j, net); `attack`
 * holds the fields of rcmarl_tailored_attack_job with their meaning there.  All arithmetic is fp32 (DnC's centring and
 * eigen-solve fp64, as in rcmarl_dnc_aggregate); every operation marked (+) (-) (*) (/) is rounded on its own, no FMA.
 *   Step.    step_k(x) is rcmarl_momentum_mix's arithmetic for slot k (the same device code): u = x (-) c, M'_k = u if
 *            first or where M_k is finite and u is not, M_k where M_k is +-inf, beta (*) M_k (+) (1 (-) beta) (*) u
 *            elsewhere; step_k(x) = c (+) M'_k.  M is read only when first = 0.
 *   Rows.    A real slot k has the row r_k = step_k(x_k) of its message x_k.  mu, d and gamma_mm are those of
 *            rcmarl_tailored_attack (the same device code and summation orders) over the honest slots' rows r_k in slot
 *            order (repeats count), and so are Gamma = scale * gamma_mm, the K + 1 candidates gamma_i and the targets
 *            t_i = m(gamma_i).
 *   Inversion.  The message that puts slot k's row at t: inv_k(t)_p = t_p if first or M_k,p is +-inf, else
 *              c_p (+) (((t_p (-) c_p) (-) (beta (*) M_k,p)) (/) (1 (-) beta)).
 *            The own slots (own_mask) all receive inv_k0(t_i), k0 the lowest own slot; every other crafted slot k is a
 *            colluder, modelled as sending inv_k(t_i) with its own state.  Crafted slot k's modelled row is
 *            a_k = step_k(the message it receives): the row j computes, not t_i.  A candidate is infeasible if one of
 *            these crafted messages has a coordinate that is not finite: O_i = -inf.
 *   Rule.    j's rule reads the n_in rows (r_k of the real slots, a_k of the crafted ones; own = row 0) with H: family
 *            COORD resilient_mean per coordinate (rcmarl_consensus_hidden's arithmetic), VECTOR exactly
 *            rcmarl_vector_aggregate's output, SPECTRAL (rule RCMARL_SPECTRAL_DNC) exactly rcmarl_dnc_aggregate's.
 *   Objective.  O_i = sum_p (R(gamma_i)_p - mu_p)^2 as in rcmarl_tailored_attack (-inf if not finite), against the
 *            honest rows' mu; i* = argmax_i O_i, ties to the smaller i, i* = 0 if every O_i is -inf.
 *   Output.  dst[0:n] = inv_k0(t_i*), gamma_out (optional, one float) = gamma_i*, model_out (optional, n floats) =
 *            R(gamma_i*): the receiver's aggregate as the attacker models it.  momentum and ref are never written.
 * Exactness: when every colluder occupies one slot of j and runs a job with the same parameters, model_out is bitwise
 * what j computes from the messages actually sent -- rcmarl_momentum_mix, then rcmarl_consensus_hidden over all n
 * parameters (COORD; for the hidden layers exact only when j combines its head through rcmarl_team, as for the
 * tailored attack), rcmarl_vector_aggregate (VECTOR) or rcmarl_dnc_aggregate (SPECTRAL).  With c = 0, first = 1,
 * inputs free of -0 and finite targets, every row is the raw message and dst, gamma_out and model_out are bitwise those
 * of rcmarl_pipeline_attack with mixing none.  NaN inputs are not supported.
 * One CTA per job: the real slots' rows, mu, d, the target, the output row, one row per crafted slot and (DnC) the fp64
 * mean staged in shared memory; the crafted slots' M rows are read from global memory for each candidate.  Fixed
 * summation orders, no atomics -- bitwise reproducible, independent of the job order and of how jobs are split over
 * launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst, gamma_out and model_out untouched): everything rcmarl_tailored_attack
 * refuses (family SPECTRAL with rule RCMARL_SPECTRAL_DNC excepted), a null ref or momentum, a beta that is not finite or
 * lies outside [0, 1), first other than 0 or 1, an own_mask that is empty or has a bit on a real slot or at or past
 * n_in, a staging size (n_in + 4 + (DnC ? 2 : 0)) * n above RCMARL_HISTORY_MAX_FLOATS (the bound admits the 16-agent
 * team-reward net, 1421 parameters, at n_in = 16 under DnC), a written range (dst, gamma_out, model_out) that overlaps
 * a real slot's row, a ref or one of the n_in M rows of any job of the launch, and two written ranges of the launch
 * that overlap. */
#define RCMARL_HISTORY_MAX_FLOATS (22 * 1421)
typedef struct {
    rcmarl_tailored_attack_job attack;   /* family COORD, VECTOR or SPECTRAL; slots, H and dev as for the tailored attack */
    float* model_out;           /* optional [n]: R(gamma_i*), the receiver's aggregate as the attacker models it */
    const float* ref;           /* [n]: c, the receiver's net after its previous consensus step */
    const float* momentum;      /* n_in rows at momentum + k * momentum_stride: the receiver's M, read only */
    int64_t momentum_stride;
    float beta;                 /* 0 <= beta < 1 */
    int32_t first;              /* 1: the receiver's first momentum step (M not read) */
    uint32_t own_mask;          /* bit k: crafted slot k receives this job's dst */
    int32_t reserved;
} rcmarl_history_attack_job;
int rcmarl_history_attack(const rcmarl_history_attack_job* jobs_host, int n_jobs, void* stream);

/* ARC-aware Byzantine messages (rcmarl_pipeline_arc_attack, rcmarl_history_arc_attack): the pipeline and history attacks
 * against a receiver j that clips (rcmarl_arc_clip) before its mixing step and rule.  Threat model: that of the base
 * attack, plus j's clipping step, whose only parameter is the job's H.  The jobs are rcmarl_pipeline_attack_job and
 * rcmarl_history_attack_job with every field's meaning unchanged; ARC runs on the rows the base attack hands on:
 *   rcmarl_pipeline_arc_attack   the slot list x(gamma_i), before the mixing step (received -> ARC -> [nnm | bucket]
 *                                -> rule);
 *   rcmarl_history_arc_attack    the momentum rows (r_k of the real slots, a_k of the crafted ones), before the rule
 *                                (received -> momentum -> ARC -> rule).
 *   ARC.     For each candidate gamma_i, rcmarl_arc_clip's arithmetic bit for bit over those n_in rows y_k (y_0 = row 0,
 *            the receiver's own, which must be real): d_k = sqrtf(the squared distance of y_k and y_0, summed as in
 *            rcmarl_arc_clip), k_clip = (2 * H * (n_in - H)) / n_in, tau and c_k by its rank rule (the same device code);
 *            the clipped row k is y_k bitwise if c_k = 1, y_0 bitwise if c_k = 0, else y_0,p + c_k * (y_k,p - y_0,p)
 *            with every operation rounded on its own.  The mixing step (or, without mixing, the rule) reads the clipped
 *            rows in place of the y_k.  The real slots' d_k do not depend on gamma_i and are taken once per job; under
 *            bucketing ARC runs once per candidate, before the n_perms shuffle samples.
 *   Everything else is the base attack's: mu, d and gamma_mm over the honest rows before ARC (the raw messages in the
 *   pipeline form, the momentum rows in the history form), O_i = sum_p (R(gamma_i)_p - mu_p)^2, the pick, dst and
 *   gamma_out; model_out = R(gamma_i*) (R_0 under bucketing) taken through ARC.
 * At H = 0 (k_clip = 0) with finite rows, ARC is the identity, so dst, gamma_out and model_out are bitwise those of the
 * base attack.  Exactness: under the base attack's conditions, model_out is bitwise what j computes from the messages
 * actually sent -- [rcmarl_momentum_mix] -> rcmarl_arc_clip -> [rcmarl_nnm_mix] -> rcmarl_consensus_hidden over all n
 * parameters (COORD), rcmarl_vector_aggregate (VECTOR) or rcmarl_dnc_aggregate (SPECTRAL); under bucketing, with the
 * attacker's sample 0 in place of j's secret shuffle.  +-inf or 1e30 real rows get c_k = 0 (they become y_0), as in
 * rcmarl_arc_clip.  NaN inputs are not supported.  One CTA per job: the clipped rows (at most k_clip of them) are staged
 * in shared memory behind the base attack's staging; fixed summation orders, no atomics -- bitwise reproducible,
 * independent of the job order and of how jobs are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst, gamma_out and model_out untouched): everything the base entry point
 * refuses, a crafted slot 0, and a job whose base staging size plus k_clip * n floats exceeds the base bound
 * (RCMARL_PIPELINE_MAX_FLOATS / RCMARL_HISTORY_MAX_FLOATS).  At the 16-agent team-reward net (1421 parameters) with
 * n_in = 16 and 15 real slots, those bounds admit: the pipeline form without mixing, and under bucketing with s >= 2,
 * every H; under bucketing with s = 1 k_clip <= 3 (H <= 2) without DnC and k_clip <= 1 (H = 1) with DnC; under nnm
 * k_clip <= 2 (H = 1) without DnC and no H >= 1 with DnC.  The history form: k_clip <= 2 (H = 1) without DnC and no
 * H >= 1 with DnC.  Every shape of the 5-agent team (n_in <= 5, at most 761 parameters) is admitted. */
int rcmarl_pipeline_arc_attack(const rcmarl_pipeline_attack_job* jobs_host, int n_jobs, void* stream);
int rcmarl_history_arc_attack(const rcmarl_history_attack_job* jobs_host, int n_jobs, void* stream);

/* Subset-aware Byzantine messages (rcmarl_subset_pipeline_attack, rcmarl_subset_history_attack): the pipeline and
 * history attacks, with or without ARC, against a receiver j whose rule is exact subset selection (MDA or SMEA,
 * rcmarl_subset_aggregate).  Threat model: that of the base attack, plus j's rule.  The jobs are
 * rcmarl_pipeline_attack_job and rcmarl_history_attack_job with every field's meaning unchanged, except that the family
 * is RCMARL_TAILOR_SUBSET and the rule an rcmarl_subset_rule:
 *   rcmarl_subset_pipeline_attack   received -> [ARC] -> [nnm | bucket] -> MDA / SMEA (the pipeline form; arc = 1:
 *                                   rcmarl_pipeline_arc_attack's clipping step);
 *   rcmarl_subset_history_attack    received -> momentum -> [ARC] -> MDA / SMEA (the history form; arc = 1:
 *                                   rcmarl_history_arc_attack's clipping step).
 *   Rule.    For each candidate gamma_i (and each shuffle sample q under bucketing), rcmarl_subset_aggregate's arithmetic
 *            bit for bit over the n_rows rows the base attack's rule reads, at H (the same device code): the flagged
 *            set F, the fp64 distances (one warp per pair, the fixed xor butterfly), the s-subsets of U in
 *            lexicographic rank order, MDA's diameter or SMEA's lambda_max(B_S) by warp_jacobi, S* = argmin c(S) with
 *            ties to the lower rank, and the fp32 mean of S* summed from 0.  The flags and pairwise distances of rows
 *            that do not depend on gamma_i (the real slots in the pipeline form without mixing or ARC and in the
 *            history form without ARC) are taken once per job by the same warp code; every other distance is summed
 *            per candidate.  No subset is skipped.
 *   Everything else is the base attack's: mu, d, Gamma, the K + 1 candidates, O_i, the pick, dst, gamma_out and
 *   model_out = R(gamma_i*) (R_0 under bucketing), with ARC (arc = 1) exactly where the ARC forms put it.
 * At H = 0 with finite rows, the rule is the plain mean, bitwise rcmarl_dnc_aggregate's at H = 0, so dst, gamma_out and
 * model_out are bitwise those of the base entry point with family SPECTRAL (DnC) at H = 0 (rcmarl_pipeline_attack,
 * rcmarl_history_attack, or their ARC forms when arc = 1).  Exactness: under the base attack's conditions, model_out is
 * bitwise what j computes from the messages actually sent -- [rcmarl_momentum_mix] -> [rcmarl_arc_clip] ->
 * [rcmarl_nnm_mix] -> rcmarl_subset_aggregate; under bucketing, with the attacker's sample 0 in place of j's secret
 * shuffle.  NaN inputs are not supported.  Each candidate runs a full subset search, up to C(16, 8) = 12 870 subsets:
 * at n_in = 16 and H >= 5 under SMEA a job takes seconds.  One CTA per job, the staging of the base attack (no fp64
 * mean) in shared memory; fixed summation orders, no atomics -- bitwise reproducible, independent of the job order and
 * of how jobs are split over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst, gamma_out and model_out untouched): everything the base entry point
 * (arc = 1: its ARC form) refuses except the family -- a family other than RCMARL_TAILOR_SUBSET, a rule other than
 * RCMARL_SUBSET_MDA and RCMARL_SUBSET_SMEA, H outside [0, n_rows) -- arc other than 0 or 1, with arc = 1 a crafted slot
 * 0, and a staging size above RCMARL_SUBSET_ATTACK_MAX_FLOATS: (n_real + n_mixed + 4 + k_clip) * n in the pipeline form
 * and (n_in + 4 + k_clip) * n in the history form (n_real, n_mixed as for rcmarl_pipeline_attack; k_clip =
 * (2 * H * (n_in - H)) / n_in with arc = 1, else 0).  The bound admits every shape of the 5-agent team (n_in <= 5, at
 * most 761 parameters) in all four forms and, at the 16-agent team-reward net (1421 parameters) with n_in = 16 and 15
 * real slots: the pipeline form without mixing (19 rows) and under bucketing with s >= 2 (at most 27 rows), with ARC at
 * every H (k_clip <= 8); under bucketing with s = 1 (34 rows) with ARC at H <= 1; under nnm (35 rows) without ARC
 * (with ARC at H = 0 only); the history form (20 rows), with ARC at every H (at most 28 rows).  Static shared memory
 * plus the bound stays under the 227 KB a CTA may opt in to (ptxas -v: at most 27 760 bytes static). */
#define RCMARL_SUBSET_ATTACK_MAX_FLOATS (35 * 1421)
int rcmarl_subset_pipeline_attack(const rcmarl_pipeline_attack_job* jobs_host, int n_jobs, int arc, void* stream);
int rcmarl_subset_history_attack(const rcmarl_history_attack_job* jobs_host, int n_jobs, int arc, void* stream);

/* IOS-aware Byzantine messages (rcmarl_ios_pipeline_attack, rcmarl_ios_history_attack): the pipeline and history
 * attacks, with or without ARC, against a receiver j whose rule is the iterative outlier scissor (rcmarl_ios_aggregate).
 * Threat model: that of the base attack, plus j's rule.  The jobs are rcmarl_pipeline_attack_job and
 * rcmarl_history_attack_job with every field's meaning unchanged, except that the family is RCMARL_TAILOR_FILTER and the
 * rule an rcmarl_filter_rule:
 *   rcmarl_ios_pipeline_attack   received -> [ARC] -> [nnm | bucket] -> IOS (the pipeline form; arc = 1:
 *                                rcmarl_pipeline_arc_attack's clipping step);
 *   rcmarl_ios_history_attack    received -> momentum -> [ARC] -> IOS (the history form; arc = 1:
 *                                rcmarl_history_arc_attack's clipping step).
 *   Rule.    For each candidate gamma_i (and each shuffle sample q under bucketing), rcmarl_ios_aggregate's arithmetic
 *            bit for bit over the n_rows rows the base attack's rule reads, at H (the same device code): the flagged
 *            set F, max(0, H - |F|) removals, each with the fp64 centre from scratch (staged, as DnC's mean, in front of
 *            the real slots), the fp64 d_k (one warp per row, the fixed xor butterfly) and the argmax removed (equal d:
 *            the higher index first, so of colluding crafted slots, whose rows are bitwise equal, the highest goes
 *            first), then the fp32 mean of the rows left, summed from 0.  Every candidate runs the full loop.
 *   Everything else is the base attack's: mu, d, Gamma, the K + 1 candidates, O_i, the pick, dst, gamma_out and
 *   model_out = R(gamma_i*) (under bucketing R_0, with the attacker's sample 0), with ARC (arc = 1) exactly where the ARC
 *   forms put it.
 * At H = 0 with finite rows, the rule is the plain mean, bitwise rcmarl_dnc_aggregate's at H = 0, so dst, gamma_out and
 * model_out are bitwise those of the base entry point with family SPECTRAL (DnC) at H = 0 (rcmarl_pipeline_attack,
 * rcmarl_history_attack, or their ARC forms when arc = 1).  Exactness: under the base attack's conditions, model_out is
 * bitwise what j computes from the messages actually sent -- [rcmarl_momentum_mix] -> [rcmarl_arc_clip] ->
 * [rcmarl_nnm_mix] -> rcmarl_ios_aggregate; under bucketing, with the attacker's sample 0 in place of j's secret
 * shuffle.  NaN inputs are not supported.  One CTA per job, exactly the staging of the DnC form (the real slots, mu, d,
 * the candidate, the output row, the mixed or crafted rows, the clipped rows and the fp64 centre) in shared memory;
 * fixed summation orders, no atomics -- bitwise reproducible, independent of the job order and of how jobs are split
 * over launches.
 * Refused (RCMARL_ERR_ARG, nothing launched, dst, gamma_out and model_out untouched): everything the base entry point
 * (arc = 1: its ARC form) refuses except the family -- a family other than RCMARL_TAILOR_FILTER, a rule other than
 * RCMARL_FILTER_IOS, H outside [0, n_rows) -- arc other than 0 or 1, with arc = 1 a crafted slot 0, and a staging size
 * (n_real + n_mixed + 6 + k_clip) * n above RCMARL_PIPELINE_MAX_FLOATS in the pipeline form and (n_in + 6 + k_clip) * n
 * above RCMARL_HISTORY_MAX_FLOATS in the history form (n_real, n_mixed as for rcmarl_pipeline_attack; k_clip =
 * (2 * H * (n_in - H)) / n_in with arc = 1, else 0): the DnC form's staging under the base bounds, so the IOS forms
 * admit exactly the shapes the DnC forms admit.  At the 16-agent team-reward net (1421 parameters) with n_in = 16 and
 * 15 real slots: the pipeline form without mixing, and under bucketing with s >= 2, at every H with or without ARC;
 * under bucketing with s = 1 without ARC, and with ARC k_clip <= 1 (H = 1); under nnm without ARC, and with ARC no
 * H >= 1; the history form without ARC, and with ARC no H >= 1.  Every shape of the 5-agent team (n_in <= 5, at most
 * 761 parameters) is admitted in all four forms.  Static shared memory plus the bound stays under the 227 KB a CTA may
 * opt in to. */
int rcmarl_ios_pipeline_attack(const rcmarl_pipeline_attack_job* jobs_host, int n_jobs, int arc, void* stream);
int rcmarl_ios_history_attack(const rcmarl_history_attack_job* jobs_host, int n_jobs, int arc, void* stream);

/* ---------------------------------------------------------------------------
 * K1 / K3.  Batched forward values:  out[row] = add_scale * add[row*add_stride + add_off]
 *                                              + sum_t scale_t * net_t(x_kind_t(row))
 * Replaces critic(ns) / critic(s) / TR(sa) eager calls:
 *   TD target  r + gamma*V(ns)            agents/resilient_CAC_agents.py:114-115, adversarial:131-132,148-149
 *   TD error   TR(sa)+gamma*V(ns)-V(s)    agents/resilient_CAC_agents.py:95-98,  adversarial:113-115
 *   critic(state) logging                 training/train_agents.py:62
 * n_out == RCMARL_N_ACTIONS with `softmax` != 0 gives actor.predict (:215): out[row][5]. */
typedef struct {
    const float* w[RCMARL_MAX_TERMS];
    int32_t kind[RCMARL_MAX_TERMS];
    float scale[RCMARL_MAX_TERMS];
    int32_t n_terms;
    int32_t n_out;              /* 1, or RCMARL_N_ACTIONS (single term only) */
    int32_t softmax;
    int32_t add_off;
    const float* add;           /* optional [rows*add_stride] indexed by absolute buffer row */
    int64_t add_stride;
    float add_scale;
    float* out;                 /* indexed by absolute buffer row */
} rcmarl_value_job;
int rcmarl_values(const rcmarl_rows* rows_host, const rcmarl_value_job* jobs_host, int n_jobs,
                  void* stream);

/* ---------------------------------------------------------------------------
 * K2 / K7 / K9.  Gradient of a summed loss over a row set, for many networks at once.
 *   mode RCMARL_LOSS_MSE:  sum_rows (net(x) - target[row])^2      (Keras MSE * B)
 *   mode RCMARL_LOSS_CE :  sum_rows target[row] * (-log softmax(net(s))[a_row])
 *                          with a_row = sa[row][3*action_agent+2] (Keras weighted sparse CE * B)
 * sums[j] = [ d(loss)/d(theta) (n_params) | loss ]   -- UNSCALED sums, so that a data-parallel
 * all-reduce can be applied before the division by the global batch size.
 * Replaces the forward/backward inside critic.fit / TR.fit / actor.train_on_batch / actor.fit
 * (agents/resilient_CAC_agents.py:99,118,136; adversarial:41,116,133,150,163,224,239,251). */
typedef enum { RCMARL_LOSS_MSE = 0, RCMARL_LOSS_CE = 1 } rcmarl_loss;
typedef struct {
    const float* w;
    const float* target;        /* regression target / TD-error weight of absolute buffer row `row`:
                                   target[row * target_stride]  (e.g. r + i with stride n_agents) */
    float* sums;                /* [n_params + 1] */
    const int32_t* time_idx;    /* optional per-job override of rows.time_idx (independent fit shuffles) */
    int64_t target_stride;
    int32_t kind;
    int32_t action_agent;       /* CE only */
} rcmarl_grad_job;
int rcmarl_grad(const rcmarl_rows* rows_host, const rcmarl_grad_job* jobs_host, int n_jobs,
                int loss_mode, void* ws, int64_t ws_bytes, void* stream);

/* theta_dst = theta_src - coef * g   (plain SGD, Keras SGD(lr): coef = lr * 2/B for MSE)
 * loss_out (optional) = loss_coef * g[n]  -- history['loss'][0] bookkeeping. */
typedef struct {
    float* dst;
    const float* src;
    const float* sums;          /* [n - first + 1]: sums for parameters [first, n) then the loss term
                                   (rcmarl_grad: first = 0;  rcmarl_team: first = n - 21) */
    float* loss_out;
    int32_t n;
    int32_t first;              /* only the parameters [first, n) are updated (frozen hidden layers, A.4) */
    float coef;
    float loss_coef;
    int32_t loss_accumulate;    /* 0: *loss_out = loss_coef*g[n];  1: *loss_out += ... (mini-batch epochs) */
    int32_t reserved;
} rcmarl_sgd_job;
int rcmarl_sgd_apply(const rcmarl_sgd_job* jobs_host, int n_jobs, void* stream);

/* K9.  Mini-batch SGD epochs for several networks (chains) in lock-step (Keras fit(batch_size=32, epochs=10,
 * shuffle=True), agents/adversarial_CAC_agents.py:133,150,163,239,251): for e < epochs, for each batch b of `mb_times`
 * time rows: rows = { time_idx_j[e*n_times + b*mb_times + i]*n_envs + env }, MSE gradient g over them (as rcmarl_grad),
 * then theta_j -= lr_j*2/(rows in batch, summed over ranks) * g in place.
 * ONE persistent kernel (csrc/minibatch_persist.cuh): the CTAs stay resident for all epochs x mini-batches, every chain's
 * parameters live in the shared memory of its CTAs, and the per-step reduction over CTAs (and, with a bound exchange
 * context, over ranks through NVLink peer memory) runs through {value, sequence} cells instead of kernel boundaries --
 * no launches, no grid barrier, no atomics; results are bitwise reproducible and identical on every rank.  Without a
 * bound exchange context a data-parallel caller loops over rcmarl_grad / all-reduce / rcmarl_sgd_apply instead.
 *   gjobs[j].time_idx: that chain's [epochs][n_times] permutation table; rows->n_rows / time_idx are ignored;
 *   sjobs[j].dst == src == gjobs[j].w, sjobs[j].n = its parameter count, sjobs[j].first = 0;
 *   sjobs[j].coef > 0 is chain j's learning rate lr_j (per-agent fast_lr, agents/resilient_CAC_agents.py:36),
 *     otherwise lr_j = `lr`;
 *   sjobs[j].loss_out (optional) receives loss_coef * sum(e^2) over epoch 0 only (history['loss'][0]), added to it
 *     when loss_accumulate;
 *   cells / cells_bytes: caller-owned scratch of rcmarl_minibatch_cells_bytes() bytes that must be ZERO before the
 *     first call and is otherwise only touched by this entry point;
 *   seq_first >= 1: first of the `rcmarl_minibatch_steps()` consecutive sequence numbers this call consumes; the
 *     caller passes strictly increasing, non-overlapping ranges over the lifetime of `cells`. */
int64_t rcmarl_minibatch_cells_bytes(int n_jobs, int max_params);
int64_t rcmarl_minibatch_steps(int epochs, int n_times, int mb_times);
int rcmarl_minibatch_fit(const rcmarl_rows* rows_host, const rcmarl_grad_job* gjobs_host,
                         const rcmarl_sgd_job* sjobs_host, int n_jobs, int epochs, int n_times, int mb_times,
                         float lr, void* cells, int64_t cells_bytes, uint32_t seq_first, void* stream);

/* Keras/TF-2 Adam (SURVEY Appendix A.5): m,v updated in place, theta -= lr_t*m/(sqrt(v)+eps);
 * g = grad_scale * sums.  lr_t = lr*sqrt(1-b2^t)/(1-b1^t) is computed by the caller. */
typedef struct {
    float* theta;
    float* m;
    float* v;
    const float* sums;
    float* loss_out;
    int32_t n;
    float grad_scale;
    float lr_t;
    float beta1, beta2, eps;
    float loss_coef;
    int32_t loss_accumulate;
    int32_t reserved;
} rcmarl_adam_job;
int rcmarl_adam_apply(const rcmarl_adam_job* jobs_host, int n_jobs, void* stream);

/* ---------------------------------------------------------------------------
 * K5 + K6 fused.  Per row: phi = features(x) with the agent's (aggregated) hidden layers;
 * est_k = phi . W3_k + b3_k for each neighbour head k (own first); agg = aggregate_k(est, H, rule);
 * projection step on the agent's own output layer:
 *   sums[0:21] = sum_rows (agg - (phi.W3_own + b3_own)) * [phi;1] / (||phi||^2 + 1)
 * so that theta_out += sums / B reproduces train_on_batch with sample weights
 * 1/(2 lr (||phi||^2+1)).  Replaces resilient_consensus_critic/_TR and
 * critic_update_team/TR_update_team (agents/resilient_CAC_agents.py:60-84,168-206).
 * agg_out (optional) stores agg per absolute row; agg_in (optional) supplies it instead (msgs, n_in, H, rule unused).
 * Refused (RCMARL_ERR_ARG, nothing launched, every sums and agg_out untouched): a null rows, sa, ns or r, n_rows < 0,
 * n_envs < 1, n_agents other than 5 and 16, a time_idx with n_rows not a multiple of n_envs, a null jobs, n_jobs outside
 * 1..RCMARL_MAX_JOBS, a null w, an unknown kind, a job with neither sums nor agg_out; for a job without agg_in also a
 * null msgs, n_in outside 1..RCMARL_MAX_NEIGHBOURS, a negative in-node, H outside [0, n_in), an unknown rule, TRIM with
 * 2H >= n_in.  A job with sums and a null or too small ws gives RCMARL_ERR_WORKSPACE. */
typedef struct {
    const float* w;             /* agent's network: aggregated hidden + current own head */
    const float* msgs;          /* message stack base (heads are read at the W3/b3 offsets) */
    int64_t msg_stride;
    float* sums;                /* [21 + 1] : projection numerators | sum (agg-pred)^2 * weight */
    float* agg_out;
    const float* agg_in;
    int32_t kind;
    int32_t n_in;
    int32_t H;
    int32_t in_nodes[RCMARL_MAX_NEIGHBOURS];
    int32_t rule;               /* rcmarl_agg_rule; 0 (a zero-initialised job) is CLIP */
} rcmarl_team_job;
int rcmarl_team(const rcmarl_rows* rows_host, const rcmarl_team_job* jobs_host, int n_jobs,
                void* ws, int64_t ws_bytes, void* stream);

/* out[row] = scale * sum over listed agents of r[row][i] / n_listed, accumulated in list order
 * (r_coop, training/train_agents.py:96-98; scale = -1 gives the Malicious agent's -r_coop, :115-116). */
int rcmarl_reward_mix(const float* r, int64_t n_rows, int n_agents, const int32_t* agents_host,
                      int n_listed, float scale, float* out, void* stream);

/* ---------------------------------------------------------------------------
 * Data parallelism over environment shards (SURVEY 8e): one process per GPU of ONE node.  A bound exchange context
 * makes rcmarl_grad / rcmarl_team return, and rcmarl_minibatch_fit apply, sums over ALL ranks: the per-CTA partials
 * are reduced, exchanged through NVLink peer memory (CUDA IPC buffers, one-shot all-reduce, rank-ordered summation =>
 * bitwise identical results on every rank) and, for the mini-batch fit, applied -- all inside ONE kernel
 * (csrc/comm.cuh).  Every rank must issue the same sequence of those calls.  Without a bound context the caller
 * all-reduces `sums` itself (e.g. NCCL) between rcmarl_grad and the apply.
 *   create(rank, world <= 8, capacity) -> export a 64-byte IPC handle -> exchange handles out of band (e.g.
 *   torch.distributed.all_gather_object) -> connect(all handles, rank-major) -> bind. */
int rcmarl_comm_create(int rank, int world, int64_t max_floats, void** comm_out);
int rcmarl_comm_handle_bytes(void);
int rcmarl_comm_export(void* comm, void* handle_out_host);
int rcmarl_comm_connect(void* comm, const void* handles_host);
int rcmarl_comm_bind(void* comm);                /* NULL unbinds */
int rcmarl_comm_error(void* comm);               /* 1 if a peer wait timed out (synchronises the device) */
int rcmarl_comm_destroy(void* comm);

/* ---------------------------------------------------------------------------
 * K1 + K8.  A block of episodes under a fixed policy for n_envs environments
 * (training/train_agents.py:46-80 + environments/grid_world.py:37-72 +
 * get_action, agents/resilient_CAC_agents.py:208-219): one thread per (episode, env).
 * Randomness, unless injected through `uniforms` / `init_state` (parity tests): Philox4x32-10 (Salmon et al. 2011,
 * the generator of rcmarl_attack) with key (seed low word, seed high word).  With g = env_offset + env (64 bits),
 * ep = the low 32 bits of episode_offset + episode, NA = n_agents (the 5- or 16-agent instantiation, also when
 * n_active is smaller), j = step, i = agent < n_active, and u01(w) = (w >> 8) * 2^-24 (exact in fp32, in [0, 1)):
 *   reset   counter (g low, g high ^ 0x80000000, ep, i)  -> (x, y, ., .):  px = umulhi(x, nrow) = (x * nrow) >> 32,
 *                                                                           py = umulhi(y, ncol)
 *   action  counter (g low, g high, ep, j * NA + i)      -> (x, y, z, .):  u0 = u01(x), u1 = u01(y), u2 = u01(z)
 * and get_action takes random_action = min(floor(u0 * 5), 4), the policy action = #{o : cdf_o / cdf_4 <= u1} (capped
 * at 4, cdf in fp32), and the policy action if u2 < 1 - mu, else the random one.  Word 1 keeps the streams apart: bit
 * 31 is set in every reset counter and clear in every action counter, and rcmarl_attack's word 1 (attacker | receiver
 * << 8 | 0x40000000) has bit 31 clear and bit 30 set, rcmarl_bucket_mix's (receiver | net << 8 | 0x20000000) bits 31
 * and 30 clear and bit 29 set, and rcmarl_pipeline_attack's (attacker | receiver << 8 | net << 16 | 0x10000000) bits
 * 31 to 29 clear and bit 28 set, so while g < 2^60 no two of the five streams share a counter.
 * Within a stream the counters are distinct while j * NA + i < 2^32; the episode word repeats after 2^32 episodes.
 * An injected `uniforms` / `init_state` replaces the draws one for one, laid out [episode][step][env][n_active][3] and
 * [episode][env][n_active][2]. */
typedef struct {
    const float* actor_w;       /* [n_agents][P_actor] */
    const float* critic_w;      /* [n_agents][P_critic] for the est_returns log (train_agents.py:62) */
    const int32_t* desired;     /* [n_agents][2] */
    float* sa; float* ns; float* r;     /* buffer bases */
    int64_t time_begin;         /* first time row written */
    float* est;                 /* [n_episodes][n_envs][n_agents] critic(state_0) */
    float* ret;                 /* [n_episodes][n_envs][n_agents] discounted returns */
    const float* uniforms;      /* optional [n_episodes][max_ep_len][n_envs][n_agents][3] */
    const int32_t* init_state;  /* optional [n_episodes][n_envs][n_agents][2] */
    uint64_t seed;
    int64_t env_offset;         /* global index of local env 0 (data-parallel shards) */
    int64_t episode_offset;
    int32_t n_envs, n_agents, n_episodes, max_ep_len;
    int32_t nrow, ncol;
    float gamma, mu;
    int32_t n_active;           /* agents 0 .. n_active-1 exist (main.py:26 --n_agents); the remaining slots of the
                                   5- / 16-agent instantiation are written as zeros.  0 means n_agents. */
    int32_t reserved;
    float state_tab_x[RCMARL_MAX_GRID];   /* (i-mean)/std, rounded from float64 by the host */
    float state_tab_y[RCMARL_MAX_GRID];
} rcmarl_rollout_args;
int rcmarl_rollout(const rcmarl_rollout_args* args_host, void* stream);

/* Means over the environments of the per-episode logs written by rcmarl_rollout (`est`, `ret`: [n_episodes][n_envs][n_agents])
 * -> out [n_episodes][n_agents]: what training/train_agents.py:168-180 prints and stores per episode, for N environments. */
int rcmarl_episode_means(const float* x, int n_episodes, int n_envs, int n_agents, float* out, void* stream);

/* One transition of Grid_World.step + get_data for n_envs environments
 * (environments/grid_world.py:47-72): state int32 [n_envs][n_agents][2] updated in place. */
int rcmarl_env_step(int32_t* state, const float* action, const int32_t* desired, int n_envs,
                    int n_agents, int nrow, float* reward_scaled, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RCMARL_H */
