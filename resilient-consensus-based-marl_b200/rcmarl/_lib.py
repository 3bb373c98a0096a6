"""ctypes binding of librcmarl.so (C ABI declared in include/rcmarl.h).

There is deliberately NO fallback: if the shared library is missing or a call
fails, an exception is raised.  The library is built in-tree by
``__graft_entry__.build()`` / ``make -C resilient-consensus-based-marl_b200/csrc``.
"""
import ctypes as C
import math
import numbers
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# override: another build of the library, e.g. to compare two builds output by output (bench.py --dump-outputs)
LIB_PATH = os.environ.get("RCMARL_LIB", os.path.join(_HERE, "librcmarl.so"))

MAX_JOBS = 32
MAX_TERMS = 3
MAX_NEIGHBOURS = 16
MAX_H = 7
MAX_GRID = 32
HIDDEN = 20
N_ACTIONS = 5

IN_S, IN_SA, IN_NS = 0, 1, 2
LOSS_MSE, LOSS_CE = 0, 1
AGG_CLIP, AGG_TRIM, AGG_WMSR = 0, 1, 2            # rcmarl_agg_rule
AGG_RULES = {"clip": AGG_CLIP, "trim": AGG_TRIM, "wmsr": AGG_WMSR}
ATTACK_ALIE, ATTACK_IPM, ATTACK_GAUSS = 0, 1, 2   # rcmarl_attack_kind
ATTACKS = {"alie": ATTACK_ALIE, "ipm": ATTACK_IPM, "gauss": ATTACK_GAUSS}
VEC_KRUM, VEC_MKRUM, VEC_SCCLIP, VEC_GMED = 0, 1, 2, 3   # rcmarl_vector_rule
VECTOR_RULES = {"krum": VEC_KRUM, "mkrum": VEC_MKRUM, "scclip": VEC_SCCLIP, "gmed": VEC_GMED}
GMED_ITERS = 8
GMED_NU = 1e-6
VECTOR_MAX_FLOATS = 48 * 1024
ADAPT_MINMAX, ADAPT_MINSUM = 0, 1                 # rcmarl_adaptive_kind
DEV_UV, DEV_STD, DEV_SGN = 0, 1, 2                # rcmarl_adaptive_dev
# min-max / min-sum attacks (rcmarl_adaptive_attack): name -> (kind, dev); the parameter is the scale s >= 0
ADAPTIVE_ATTACKS = {f"{k}_{d}": (kind, dev) for k, kind in (("minmax", ADAPT_MINMAX), ("minsum", ADAPT_MINSUM))
                    for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}
ADAPTIVE_MAX_FLOATS = 18 * 1536
TAILOR_COORD, TAILOR_VECTOR, TAILOR_SPECTRAL, TAILOR_SUBSET, TAILOR_FILTER = 0, 1, 2, 3, 4   # rcmarl_tailored_family
# rule-aware attacks (rcmarl_tailored_attack): candidate steps K and the staging bound; the names are TAILORED_ATTACKS
TAILORED_STEPS = 32
TAILORED_MAX_FLOATS = 19 * 1536
SPECTRAL_DNC = 0                                  # rcmarl_spectral_rule
SPECTRAL_RULES = {"dnc": SPECTRAL_DNC}
DNC_SWEEPS = 32
DNC_MAX_FLOATS = 48 * 1024
SUBSET_MDA, SUBSET_SMEA = 0, 1                    # rcmarl_subset_rule
SUBSET_RULES = {"mda": SUBSET_MDA, "smea": SUBSET_SMEA}
SUBSET_MAX_FLOATS = 48 * 1024
FILTER_IOS = 0                                    # rcmarl_filter_rule
FILTER_RULES = {"ios": FILTER_IOS}
IOS_MAX_FLOATS = 48 * 1024
MIX_NNM = 0                                       # rcmarl_mixing_rule
MIXING_RULES = {"nnm": MIX_NNM}
NNM_MAX_FLOATS = 48 * 1024
MIX_BUCKET = 1                                    # rcmarl_mixing_rule: randomized bucketing, ("bucket", s)
BUCKET_DEFAULT_S = 2                              # the bucket size of a plain "bucket" entry
BUCKET_MAX_S = 2 ** 31 - 1
MIX_MOMENTUM = 2                                  # rcmarl_mixing_rule: per-neighbour momentum at beta, 0 <= beta < 1
MIX_ARC = 3                                       # rcmarl_mixing_rule: adaptive robust clipping, clipping="arc"
# pipeline-aware attacks (rcmarl_pipeline_attack): rcmarl_pipeline_mixing, the staging bound, the most shuffle samples
# and the samples the trainer draws; the names are PIPELINE_ATTACKS
PIPE_NONE, PIPE_NNM, PIPE_BUCKET = 0, 1, 2
PIPELINE_MAX_FLOATS = 37 * 1421
PIPELINE_MAX_PERMS = 16
PIPELINE_PERMS = 4
# momentum-aware attacks (rcmarl_history_attack): the staging bound; the names are HISTORY_ATTACKS
HISTORY_MAX_FLOATS = 22 * 1421
# subset-aware attacks (rcmarl_subset_pipeline_attack / rcmarl_subset_history_attack): the staging bound; the names
# are SUBSET_ATTACKS
SUBSET_ATTACK_MAX_FLOATS = 35 * 1421
MIMIC_MAX_FLOATS = 19 * 1536                      # rcmarl_mimic_attack's staging bound
MIMIC_MAX_T0 = 2 ** 31 - 1                        # the mimic attack's power steps T0: an integer in 0 .. 2^31 - 1

c_fp = C.c_void_p  # device pointers travel as integers


class Rows(C.Structure):
    _fields_ = [("sa", c_fp), ("ns", c_fp), ("r", c_fp), ("row_begin", C.c_int64), ("n_rows", C.c_int64),
                ("time_idx", c_fp), ("n_envs", C.c_int32), ("n_agents", C.c_int32)]


class ConsensusJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("n_hidden", C.c_int32),
                ("n_in", C.c_int32), ("H", C.c_int32), ("in_nodes", C.c_int32 * MAX_NEIGHBOURS), ("rule", C.c_int32)]


class AttackJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("n", C.c_int32), ("n_honest", C.c_int32),
                ("honest", C.c_int32 * MAX_NEIGHBOURS), ("kind", C.c_int32), ("param", C.c_float), ("seed", C.c_uint64),
                ("attacker", C.c_uint32), ("receiver", C.c_uint32), ("round", C.c_uint32), ("epoch", C.c_uint32)]


class VectorJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("weights_out", c_fp), ("n", C.c_int32),
                ("n_in", C.c_int32), ("H", C.c_int32), ("rule", C.c_int32), ("in_nodes", C.c_int32 * MAX_NEIGHBOURS)]


class AdaptiveAttackJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("gamma_out", c_fp), ("n", C.c_int32),
                ("n_honest", C.c_int32), ("honest", C.c_int32 * MAX_NEIGHBOURS), ("kind", C.c_int32), ("dev", C.c_int32),
                ("scale", C.c_float), ("reserved", C.c_int32)]


class TailoredAttackJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("gamma_out", c_fp), ("n", C.c_int32),
                ("n_in", C.c_int32), ("slots", C.c_int32 * MAX_NEIGHBOURS), ("honest_mask", C.c_uint32),
                ("family", C.c_int32), ("rule", C.c_int32), ("H", C.c_int32), ("dev", C.c_int32), ("scale", C.c_float)]


class PipelineAttackJob(C.Structure):
    _fields_ = [("attack", TailoredAttackJob), ("model_out", c_fp), ("seed", C.c_uint64), ("mixing", C.c_int32),
                ("s", C.c_int32), ("n_perms", C.c_int32), ("attacker", C.c_uint32), ("receiver", C.c_uint32),
                ("net", C.c_uint32), ("round", C.c_uint32), ("epoch", C.c_uint32)]


class HistoryAttackJob(C.Structure):
    _fields_ = [("attack", TailoredAttackJob), ("model_out", c_fp), ("ref", c_fp), ("momentum", c_fp),
                ("momentum_stride", C.c_int64), ("beta", C.c_float), ("first", C.c_int32), ("own_mask", C.c_uint32),
                ("reserved", C.c_int32)]


class DissensusJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("n", C.c_int32), ("own", C.c_int32),
                ("n_honest", C.c_int32), ("honest", C.c_int32 * MAX_NEIGHBOURS), ("n_byz", C.c_int32),
                ("eps", C.c_float), ("reserved", C.c_int32)]


class MimicJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("z", c_fp), ("target_out", c_fp),
                ("n", C.c_int32), ("n_honest", C.c_int32), ("honest", C.c_int32 * MAX_NEIGHBOURS),
                ("candidate_mask", C.c_uint32), ("update", C.c_int32)]


class BucketJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("weights_out", c_fp), ("n", C.c_int32),
                ("n_in", C.c_int32), ("s", C.c_int32), ("in_nodes", C.c_int32 * MAX_NEIGHBOURS), ("seed", C.c_uint64),
                ("receiver", C.c_uint32), ("net", C.c_uint32), ("round", C.c_uint32), ("epoch", C.c_uint32)]


class MomentumJob(C.Structure):
    _fields_ = [("dst", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("ref", c_fp), ("momentum", c_fp),
                ("momentum_stride", C.c_int64), ("n", C.c_int32), ("n_in", C.c_int32),
                ("in_nodes", C.c_int32 * MAX_NEIGHBOURS), ("beta", C.c_float), ("first", C.c_int32)]


class ValueJob(C.Structure):
    _fields_ = [("w", c_fp * MAX_TERMS), ("kind", C.c_int32 * MAX_TERMS), ("scale", C.c_float * MAX_TERMS),
                ("n_terms", C.c_int32), ("n_out", C.c_int32), ("softmax", C.c_int32), ("add_off", C.c_int32),
                ("add", c_fp), ("add_stride", C.c_int64), ("add_scale", C.c_float), ("out", c_fp)]


class GradJob(C.Structure):
    _fields_ = [("w", c_fp), ("target", c_fp), ("sums", c_fp), ("time_idx", c_fp), ("target_stride", C.c_int64),
                ("kind", C.c_int32), ("action_agent", C.c_int32)]


class SgdJob(C.Structure):
    _fields_ = [("dst", c_fp), ("src", c_fp), ("sums", c_fp), ("loss_out", c_fp), ("n", C.c_int32),
                ("first", C.c_int32), ("coef", C.c_float), ("loss_coef", C.c_float), ("loss_accumulate", C.c_int32),
                ("reserved", C.c_int32)]


class AdamJob(C.Structure):
    _fields_ = [("theta", c_fp), ("m", c_fp), ("v", c_fp), ("sums", c_fp), ("loss_out", c_fp), ("n", C.c_int32),
                ("grad_scale", C.c_float), ("lr_t", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float), ("loss_coef", C.c_float), ("loss_accumulate", C.c_int32), ("reserved", C.c_int32)]


class TeamJob(C.Structure):
    _fields_ = [("w", c_fp), ("msgs", c_fp), ("msg_stride", C.c_int64), ("sums", c_fp), ("agg_out", c_fp),
                ("agg_in", c_fp), ("kind", C.c_int32), ("n_in", C.c_int32), ("H", C.c_int32),
                ("in_nodes", C.c_int32 * MAX_NEIGHBOURS), ("rule", C.c_int32)]


class RolloutArgs(C.Structure):
    _fields_ = [("actor_w", c_fp), ("critic_w", c_fp), ("desired", c_fp), ("sa", c_fp), ("ns", c_fp), ("r", c_fp),
                ("time_begin", C.c_int64), ("est", c_fp), ("ret", c_fp), ("uniforms", c_fp), ("init_state", c_fp),
                ("seed", C.c_uint64), ("env_offset", C.c_int64), ("episode_offset", C.c_int64),
                ("n_envs", C.c_int32), ("n_agents", C.c_int32), ("n_episodes", C.c_int32), ("max_ep_len", C.c_int32),
                ("nrow", C.c_int32), ("ncol", C.c_int32), ("gamma", C.c_float), ("mu", C.c_float),
                ("n_active", C.c_int32), ("reserved", C.c_int32),
                ("state_tab_x", C.c_float * MAX_GRID), ("state_tab_y", C.c_float * MAX_GRID)]


# every symbol include/rcmarl.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("rcmarl_version", C.c_char_p, []),
    ("rcmarl_status_string", C.c_char_p, [C.c_int]),
    ("rcmarl_last_cuda_error", C.c_int, []),
    ("rcmarl_device_info", C.c_int, [C.POINTER(C.c_int)] * 3),
    ("rcmarl_param_count", C.c_int64, [C.c_int, C.c_int]),
    ("rcmarl_workspace_bytes", C.c_int64, [C.c_int, C.c_int]),
    ("rcmarl_grad_grid_plan", C.c_int, [C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int,
                                        C.POINTER(C.c_int32)]),
    ("rcmarl_grad_tile_map", C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int64]),
    ("rcmarl_clip_mean", C.c_int, [c_fp, C.c_int, C.c_int64, C.c_int64, C.c_int, c_fp, c_fp]),
    ("rcmarl_consensus_hidden", C.c_int, [C.POINTER(ConsensusJob), C.c_int, c_fp]),
    ("rcmarl_attack", C.c_int, [C.POINTER(AttackJob), C.c_int, c_fp]),
    ("rcmarl_vector_aggregate", C.c_int, [C.POINTER(VectorJob), C.c_int, c_fp]),
    ("rcmarl_dnc_aggregate", C.c_int, [C.POINTER(VectorJob), C.c_int, c_fp]),
    ("rcmarl_subset_aggregate", C.c_int, [C.POINTER(VectorJob), C.c_int, c_fp]),
    ("rcmarl_ios_aggregate", C.c_int, [C.POINTER(VectorJob), C.c_int, c_fp]),
    ("rcmarl_nnm_mix", C.c_int, [C.POINTER(VectorJob), C.c_int, c_fp]),
    ("rcmarl_arc_clip", C.c_int, [C.POINTER(VectorJob), C.c_int, c_fp]),
    ("rcmarl_bucket_mix", C.c_int, [C.POINTER(BucketJob), C.c_int, c_fp]),
    ("rcmarl_momentum_mix", C.c_int, [C.POINTER(MomentumJob), C.c_int, c_fp]),
    ("rcmarl_adaptive_attack", C.c_int, [C.POINTER(AdaptiveAttackJob), C.c_int, c_fp]),
    ("rcmarl_tailored_attack", C.c_int, [C.POINTER(TailoredAttackJob), C.c_int, c_fp]),
    ("rcmarl_pipeline_attack", C.c_int, [C.POINTER(PipelineAttackJob), C.c_int, c_fp]),
    ("rcmarl_history_attack", C.c_int, [C.POINTER(HistoryAttackJob), C.c_int, c_fp]),
    ("rcmarl_pipeline_arc_attack", C.c_int, [C.POINTER(PipelineAttackJob), C.c_int, c_fp]),
    ("rcmarl_history_arc_attack", C.c_int, [C.POINTER(HistoryAttackJob), C.c_int, c_fp]),
    ("rcmarl_subset_pipeline_attack", C.c_int, [C.POINTER(PipelineAttackJob), C.c_int, C.c_int, c_fp]),
    ("rcmarl_subset_history_attack", C.c_int, [C.POINTER(HistoryAttackJob), C.c_int, C.c_int, c_fp]),
    ("rcmarl_ios_pipeline_attack", C.c_int, [C.POINTER(PipelineAttackJob), C.c_int, C.c_int, c_fp]),
    ("rcmarl_ios_history_attack", C.c_int, [C.POINTER(HistoryAttackJob), C.c_int, C.c_int, c_fp]),
    ("rcmarl_dissensus_attack", C.c_int, [C.POINTER(DissensusJob), C.c_int, c_fp]),
    ("rcmarl_mimic_attack", C.c_int, [C.POINTER(MimicJob), C.c_int, c_fp]),
    ("rcmarl_values", C.c_int, [C.POINTER(Rows), C.POINTER(ValueJob), C.c_int, c_fp]),
    ("rcmarl_grad", C.c_int, [C.POINTER(Rows), C.POINTER(GradJob), C.c_int, C.c_int, c_fp, C.c_int64, c_fp]),
    ("rcmarl_sgd_apply", C.c_int, [C.POINTER(SgdJob), C.c_int, c_fp]),
    ("rcmarl_adam_apply", C.c_int, [C.POINTER(AdamJob), C.c_int, c_fp]),
    ("rcmarl_minibatch_cells_bytes", C.c_int64, [C.c_int, C.c_int]),
    ("rcmarl_minibatch_steps", C.c_int64, [C.c_int, C.c_int, C.c_int]),
    ("rcmarl_minibatch_fit", C.c_int, [C.POINTER(Rows), C.POINTER(GradJob), C.POINTER(SgdJob), C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_float, c_fp, C.c_int64, C.c_uint32, c_fp]),
    ("rcmarl_team", C.c_int, [C.POINTER(Rows), C.POINTER(TeamJob), C.c_int, c_fp, C.c_int64, c_fp]),
    ("rcmarl_reward_mix", C.c_int, [c_fp, C.c_int64, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_float, c_fp, c_fp]),
    ("rcmarl_comm_create", C.c_int, [C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_void_p)]),
    ("rcmarl_comm_handle_bytes", C.c_int, []),
    ("rcmarl_comm_export", C.c_int, [C.c_void_p, C.c_char_p]),
    ("rcmarl_comm_connect", C.c_int, [C.c_void_p, C.c_char_p]),
    ("rcmarl_comm_bind", C.c_int, [C.c_void_p]),
    ("rcmarl_comm_error", C.c_int, [C.c_void_p]),
    ("rcmarl_comm_destroy", C.c_int, [C.c_void_p]),
    ("rcmarl_rollout", C.c_int, [C.POINTER(RolloutArgs), c_fp]),
    ("rcmarl_episode_means", C.c_int, [c_fp, C.c_int, C.c_int, C.c_int, c_fp, c_fp]),
    ("rcmarl_env_step", C.c_int, [c_fp, c_fp, c_fp, C.c_int, C.c_int, C.c_int, c_fp, c_fp]),
]

_lib = None


class RcmarlError(RuntimeError):
    pass


def lib():
    """Load librcmarl.so (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RcmarlError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the RPBCAC kernels)")
        l = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            f = getattr(l, name)          # AttributeError if the ABI and the header diverge
            f.restype = res
            f.argtypes = args
        _lib = l
    return _lib


def check(status, what):
    if status != 0:
        l = lib()
        msg = l.rcmarl_status_string(status).decode()
        raise RcmarlError(f"{what}: {msg} (status {status}, cudaError {l.rcmarl_last_cuda_error()})")


def agg_rule(rule):
    """Aggregation rule name ("clip", "trim", "wmsr") or rcmarl_agg_rule id -> id.  Ids are passed through unchecked
    (the library refuses unknown ones); an unknown name raises."""
    if isinstance(rule, str):
        if rule not in AGG_RULES:
            raise RcmarlError(f"unknown aggregation rule {rule!r}: expected one of {sorted(AGG_RULES)}")
        return AGG_RULES[rule]
    return int(rule)


def check_aggregation(rule, H, n_in):
    """Raise RcmarlError unless `rule` is known and allows H trimmed values out of n_in (include/rcmarl.h): for every
    rule 1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in, for trim also 2H < n_in."""
    r = agg_rule(rule)
    if r not in AGG_RULES.values():
        raise RcmarlError(f"unknown aggregation rule id {r}")
    if not (1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in) or (r == AGG_TRIM and 2 * H >= n_in):
        raise RcmarlError(f"aggregation {rule!r} with H={H} needs 0 <= H < n_in" + (" and 2H < n_in" if r == AGG_TRIM else "")
                          + f" (n_in={n_in}, at most {MAX_NEIGHBOURS})")
    return r


def is_vector_rule(rule):
    """True for the name of a distance-based rule (rcmarl_vector_rule): "krum", "mkrum", "scclip", "gmed"."""
    return isinstance(rule, str) and rule in VECTOR_RULES


def check_vector_rule(rule, H, n_in):
    """Raise RcmarlError unless `rule` names a distance-based rule that allows H out of n_in messages
    (include/rcmarl.h): 1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in, for krum / mkrum also n_in >= H + 3.
    Returns the rcmarl_vector_rule id."""
    if not is_vector_rule(rule):
        raise RcmarlError(f"unknown distance-based aggregation rule {rule!r}: expected one of {sorted(VECTOR_RULES)}")
    krum = rule in ("krum", "mkrum")
    if not (1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in) or (krum and n_in < H + 3):
        raise RcmarlError(f"aggregation {rule!r} with H={H} needs 0 <= H < n_in" + (" and n_in >= H + 3" if krum else "")
                          + f" (n_in={n_in}, at most {MAX_NEIGHBOURS})")
    return VECTOR_RULES[rule]


def is_spectral_rule(rule):
    """True for the name of a spectral rule (rcmarl_spectral_rule): "dnc"."""
    return isinstance(rule, str) and rule in SPECTRAL_RULES


def check_spectral_rule(H, n_in):
    """Raise RcmarlError unless DnC (rcmarl_dnc_aggregate, include/rcmarl.h) allows H out of n_in messages:
    1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in.  Returns the rcmarl_spectral_rule id."""
    if not (1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in):
        raise RcmarlError(f"aggregation 'dnc' with H={H} needs 0 <= H < n_in (n_in={n_in}, at most {MAX_NEIGHBOURS})")
    return SPECTRAL_DNC


def is_subset_rule(rule):
    """True for the name of an exact subset-selection rule (rcmarl_subset_rule): "mda", "smea"."""
    return isinstance(rule, str) and rule in SUBSET_RULES


def check_subset_rule(H, n_in):
    """Raise RcmarlError unless the subset-selection rules (rcmarl_subset_aggregate, include/rcmarl.h) allow H out of
    n_in messages: 1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in.  The names are SUBSET_RULES (see is_subset_rule)."""
    if not (1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in):
        raise RcmarlError(f"aggregation 'mda' / 'smea' with H={H} needs 0 <= H < n_in (n_in={n_in}, at most "
                          f"{MAX_NEIGHBOURS})")


def is_filter_rule(rule):
    """True for the name of an iterative filtering rule (rcmarl_filter_rule): "ios"."""
    return isinstance(rule, str) and rule in FILTER_RULES


def check_filter_rule(H, n_in):
    """Raise RcmarlError unless the iterative outlier scissor (rcmarl_ios_aggregate, include/rcmarl.h) allows H out of
    n_in messages: 1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in.  Returns the rcmarl_filter_rule id."""
    if not (1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in):
        raise RcmarlError(f"aggregation 'ios' with H={H} needs 0 <= H < n_in (n_in={n_in}, at most {MAX_NEIGHBOURS})")
    return FILTER_IOS


def mixing_entry(mixing):
    """A pre-aggregation mixing entry in its stored form: None, "nnm" (rcmarl_nnm_mix) or ("bucket", s)
    (rcmarl_bucket_mix, bucket size s); "bucket" stands for ("bucket", BUCKET_DEFAULT_S).  Raise RcmarlError for
    anything else, an s that is not an integer in 1 .. BUCKET_MAX_S included."""
    if mixing is None or (isinstance(mixing, str) and mixing in MIXING_RULES):
        return mixing
    if isinstance(mixing, str) and mixing == "bucket":
        return ("bucket", BUCKET_DEFAULT_S)
    if isinstance(mixing, tuple) and len(mixing) == 2 and isinstance(mixing[0], str) and mixing[0] == "bucket":
        s = mixing[1]
        if not (isinstance(s, numbers.Integral) and not isinstance(s, bool) and 1 <= s <= BUCKET_MAX_S):
            raise RcmarlError(f"mixing 'bucket' needs an integer bucket size s in 1 .. {BUCKET_MAX_S}, got {s!r}")
        return ("bucket", int(s))
    raise RcmarlError(f"unknown mixing rule {mixing!r}: expected None or one of "
                      f"{sorted(MIXING_RULES) + ['bucket', ('bucket', 's')]}")


def is_bucket_mixing(mixing):
    """True for a bucketing entry ("bucket" or ("bucket", s)); the entry is not otherwise checked."""
    return mixing == "bucket" or (isinstance(mixing, tuple) and len(mixing) == 2 and mixing[0] == "bucket")


def check_mixing(name, H, n_in):
    """Raise RcmarlError unless `name` is a pre-aggregation mixing entry ("nnm", "bucket" or ("bucket", s), see
    mixing_entry) that allows H out of n_in messages (rcmarl_nnm_mix / rcmarl_bucket_mix, include/rcmarl.h):
    1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in.  Returns the rcmarl_mixing_rule id."""
    entry = mixing_entry(name)
    if entry is None:
        raise RcmarlError(f"unknown mixing rule {name!r}: expected None or one of "
                          f"{sorted(MIXING_RULES) + ['bucket', ('bucket', 's')]}")
    if not (1 <= n_in <= MAX_NEIGHBOURS and 0 <= H < n_in):
        raise RcmarlError(f"mixing {name!r} with H={H} needs 0 <= H < n_in (n_in={n_in}, at most {MAX_NEIGHBOURS})")
    return MIX_BUCKET if is_bucket_mixing(entry) else MIXING_RULES[entry]


def mixed_rows(mixing, n_in):
    """The number of rows an agent's rule reads after its mixing entry over n_in received messages: n_in without
    mixing and for "nnm"; 1 + ceil((n_in - 1) / s) for bucketing (the own row, then one mean per bucket)."""
    entry = mixing_entry(mixing)
    if entry is None or entry == "nnm":
        return n_in
    return 1 + -(-(n_in - 1) // entry[1])


def check_momentum(beta):
    """Raise RcmarlError unless beta is a real number that rcmarl_momentum_mix accepts (include/rcmarl.h): finite, in
    [0, 1) once rounded to fp32.  Returns it as a float."""
    if isinstance(beta, bool) or not isinstance(beta, numbers.Real):
        raise RcmarlError(f"momentum needs a real beta in [0, 1), got {beta!r}")
    b = float(C.c_float(float(beta)).value)
    if not (math.isfinite(b) and 0.0 <= b < 1.0):
        raise RcmarlError(f"momentum needs a real beta in [0, 1), got {beta!r}")
    return float(beta)


def check_clipping(name):
    """Raise RcmarlError unless `name` is a pre-aggregation clipping entry: None or "arc" (adaptive robust clipping,
    rcmarl_arc_clip).  Returns it."""
    if name is None or (isinstance(name, str) and name == "arc"):
        return name
    raise RcmarlError(f"unknown clipping {name!r}: expected None or 'arc'")


def arc_count(H, n):
    """k_clip of rcmarl_arc_clip: how many of n messages ARC may clip at H, (2 H (n - H)) // n (include/rcmarl.h)."""
    return (2 * int(H) * (int(n) - int(H))) // int(n)


def is_adaptive_attack(name):
    """True for the name of a min-max / min-sum attack (rcmarl_adaptive_attack): "minmax_uv", ..., "minsum_sgn"."""
    return isinstance(name, str) and name in ADAPTIVE_ATTACKS


class TailoredKind(int):
    """The kind check_attack gives a rule-aware attack: its rcmarl_adaptive_dev, as a type of its own so that it is
    told apart from the rcmarl_attack_kind ids and the adaptive (kind, dev) pairs."""

    def __repr__(self):
        return f"TailoredKind({int(self)})"


TAILORED_ATTACKS = {f"tailored_{d}": TailoredKind(dev) for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}


def is_tailored_attack(name):
    """True for the name of a rule-aware attack (rcmarl_tailored_attack): "tailored_uv", "tailored_std", "tailored_sgn"."""
    return isinstance(name, str) and name in TAILORED_ATTACKS


class PipelineKind(int):
    """The kind check_attack gives a pipeline-aware attack (rcmarl_pipeline_attack): its rcmarl_adaptive_dev, as a type
    of its own so that it is told apart from the tailored attacks, which model the receiver's rule only."""

    def __repr__(self):
        return f"PipelineKind({int(self)})"


PIPELINE_ATTACKS = {f"pipeline_{d}": PipelineKind(dev) for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}


def is_pipeline_attack(name):
    """True for the name of a pipeline-aware attack (rcmarl_pipeline_attack): "pipeline_uv", "pipeline_std",
    "pipeline_sgn"."""
    return isinstance(name, str) and name in PIPELINE_ATTACKS


class HistoryKind(int):
    """The kind check_attack gives a momentum-aware attack (rcmarl_history_attack): its rcmarl_adaptive_dev, as a type
    of its own so that it is told apart from the pipeline attacks, which do not model the receiver's momentum."""

    def __repr__(self):
        return f"HistoryKind({int(self)})"


HISTORY_ATTACKS = {f"history_{d}": HistoryKind(dev) for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}


def is_history_attack(name):
    """True for the name of a momentum-aware attack (rcmarl_history_attack): "history_uv", "history_std",
    "history_sgn"."""
    return isinstance(name, str) and name in HISTORY_ATTACKS


class ArcAttackKind(int):
    """The kind check_attack gives an ARC-aware attack (rcmarl_pipeline_arc_attack / rcmarl_history_arc_attack): its
    rcmarl_adaptive_dev, as a type of its own so that it is told apart from the pipeline and history attacks, which do
    not model the receiver's clipping."""

    def __repr__(self):
        return f"ArcAttackKind({int(self)})"


ARC_ATTACKS = {f"arc_{d}": ArcAttackKind(dev) for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}


def is_arc_attack(name):
    """True for the name of an ARC-aware attack: "arc_uv", "arc_std", "arc_sgn"."""
    return isinstance(name, str) and name in ARC_ATTACKS


class SubsetAttackKind(int):
    """The kind check_attack gives a subset-aware attack (rcmarl_subset_pipeline_attack / rcmarl_subset_history_attack):
    its rcmarl_adaptive_dev, as a type of its own so that it is told apart from the attacks that do not model the
    receiver's MDA / SMEA selection."""

    def __repr__(self):
        return f"SubsetAttackKind({int(self)})"


SUBSET_ATTACKS = {f"subset_{d}": SubsetAttackKind(dev) for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}


def is_subset_attack(name):
    """True for the name of a subset-aware attack: "subset_uv", "subset_std", "subset_sgn"."""
    return isinstance(name, str) and name in SUBSET_ATTACKS


class IosAttackKind(int):
    """The kind check_attack gives an IOS-aware attack (rcmarl_ios_pipeline_attack / rcmarl_ios_history_attack): its
    rcmarl_adaptive_dev, as a type of its own so that it is told apart from the attacks that do not model the
    receiver's iterative outlier scissor."""

    def __repr__(self):
        return f"IosAttackKind({int(self)})"


IOS_ATTACKS = {f"ios_{d}": IosAttackKind(dev) for d, dev in (("uv", DEV_UV), ("std", DEV_STD), ("sgn", DEV_SGN))}


def is_ios_attack(name):
    """True for the name of an IOS-aware attack: "ios_uv", "ios_std", "ios_sgn"."""
    return isinstance(name, str) and name in IOS_ATTACKS


class DissensusKind(int):
    """The kind check_attack gives the dissensus attack (rcmarl_dissensus_attack), a type of its own so that it is told
    apart from the other attacks' kinds; its parameter is eps >= 0."""

    def __repr__(self):
        return "DissensusKind()"


class MimicKind(int):
    """The kind check_attack gives the mimic attack (rcmarl_mimic_attack), a type of its own so that it is told apart
    from the other attacks' kinds; its parameter is T0, the number of power steps each (attacker, receiver) pair takes."""

    def __repr__(self):
        return "MimicKind()"


STATE_ATTACKS = {"dissensus": DissensusKind(0), "mimic": MimicKind(0)}


def check_attack(attack):
    """(name, param) -> (kind, float param); raise RcmarlError unless the name is known and the parameter finite (for
    "gauss", the adaptive, the tailored, the pipeline, the history, the ARC, the subset and the IOS attacks and
    "dissensus" also >= 0; for "mimic" an integer in 0 .. MIMIC_MAX_T0), as rcmarl_attack / rcmarl_adaptive_attack /
    rcmarl_tailored_attack / rcmarl_pipeline_attack / rcmarl_history_attack / rcmarl_pipeline_arc_attack /
    rcmarl_history_arc_attack / rcmarl_subset_pipeline_attack / rcmarl_subset_history_attack /
    rcmarl_ios_pipeline_attack / rcmarl_ios_history_attack / rcmarl_dissensus_attack / rcmarl_mimic_attack require
    (include/rcmarl.h).  kind is the rcmarl_attack_kind id of "alie", "ipm" and "gauss",
    the pair (rcmarl_adaptive_kind, rcmarl_adaptive_dev) of an adaptive attack, whose parameter is the scale s (1 is the
    paper's attack), the TailoredKind (its rcmarl_adaptive_dev) of a tailored attack, the PipelineKind of a pipeline
    attack, the HistoryKind of a history attack, the ArcAttackKind of an ARC attack, the SubsetAttackKind of a
    subset attack and the IosAttackKind of an IOS attack, whose parameter is the range multiplier s, DissensusKind for "dissensus", whose parameter is eps (1 cancels the honest pull under a plain mean),
    and MimicKind for "mimic", whose parameter is T0 (the power steps each pair takes before its direction freezes)."""
    try:
        name, param = attack
        param = float(param)
    except (TypeError, ValueError):
        raise RcmarlError(f"an attack is a (name, param) pair, got {attack!r}")
    known = {**ATTACKS, **ADAPTIVE_ATTACKS, **TAILORED_ATTACKS, **PIPELINE_ATTACKS, **HISTORY_ATTACKS, **ARC_ATTACKS,
             **SUBSET_ATTACKS, **IOS_ATTACKS, **STATE_ATTACKS}
    if not isinstance(name, str) or name not in known:
        names = sorted(ATTACKS) + sorted(ADAPTIVE_ATTACKS) + sorted(TAILORED_ATTACKS) + sorted(PIPELINE_ATTACKS) \
            + sorted(HISTORY_ATTACKS) + sorted(ARC_ATTACKS) + sorted(SUBSET_ATTACKS) + sorted(IOS_ATTACKS) \
            + sorted(STATE_ATTACKS)
        raise RcmarlError(f"unknown attack {name!r}: expected one of {names}")
    if name == "mimic":
        if not (math.isfinite(param) and param == int(param) and 0 <= param <= MIMIC_MAX_T0):
            raise RcmarlError(f"attack 'mimic' needs an integer T0 in 0 .. {MIMIC_MAX_T0}, got {param}")
        return known[name], param
    nonneg = name in ("gauss", "dissensus") or name in ADAPTIVE_ATTACKS or name in TAILORED_ATTACKS \
        or name in PIPELINE_ATTACKS or name in HISTORY_ATTACKS or name in ARC_ATTACKS or name in SUBSET_ATTACKS \
        or name in IOS_ATTACKS
    if not math.isfinite(param) or (nonneg and param < 0):
        raise RcmarlError(f"attack {name!r} needs a finite parameter" + (" >= 0" if nonneg else "") + f", got {param}")
    return known[name], param


def param_count(d_in, n_out):
    return d_in * HIDDEN + HIDDEN + HIDDEN * HIDDEN + HIDDEN + HIDDEN * n_out + n_out
