"""Thin Python wrappers over the C ABI (include/rcmarl.h): torch tensors in,
kernel launches on torch's current CUDA stream out.  PyTorch is plumbing only
(device memory, streams); every arithmetic step of the hot path happens in
librcmarl.so."""
import ctypes as C

import numpy as np
import torch

from . import _lib as L

_ws = {}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def dev_f32(x, device=None):
    """numpy / torch (any device) -> contiguous float32 CUDA tensor."""
    if isinstance(x, torch.Tensor):
        t = x
    else:
        if hasattr(x, "_t"):                       # facade Tensor
            t = x._t
        else:
            t = torch.as_tensor(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return t.to(device=device, dtype=torch.float32).contiguous()


def workspace(n_jobs=L.MAX_JOBS, max_params=None):
    """Persistent scratch for the *_grad / team entry points (caller-owned, no hidden allocation)."""
    dev = torch.cuda.current_device()
    if max_params is None:
        max_params = L.param_count(48, 1)
    need = L.lib().rcmarl_workspace_bytes(n_jobs, max_params)
    w = _ws.get(dev)
    if w is None or w.numel() < need:
        w = torch.empty(need, dtype=torch.uint8, device=f"cuda:{dev}")
        _ws[dev] = w
    return w


def make_rows(sa, ns, r, n_agents, row_begin=0, n_rows=None, time_idx=None, n_envs=1):
    """Build an rcmarl_rows.  Unused arrays may be None (a valid dummy pointer is passed)."""
    some = sa if sa is not None else (ns if ns is not None else r)
    R = L.Rows()
    R.sa = ptr(sa if sa is not None else some)
    R.ns = ptr(ns if ns is not None else some)
    R.r = ptr(r if r is not None else some)
    R.row_begin = int(row_begin)
    if n_rows is None:
        n_rows = (time_idx.numel() * n_envs) if time_idx is not None else some.shape[0]
    R.n_rows = int(n_rows)
    R.time_idx = ptr(time_idx)
    R.n_envs = int(n_envs)
    R.n_agents = int(n_agents)
    R._keep = (sa, ns, r, time_idx)
    return R


def clip_mean(vals, H, out=None):
    """vals: [n, P] float32 CUDA (row stride = vals.stride(0)); own = row 0."""
    n, P = vals.shape
    assert vals.stride(1) == 1
    if out is None:
        out = torch.empty(P, dtype=torch.float32, device=vals.device)
    if not (0 <= int(H) < n):
        raise L.RcmarlError(f"rcmarl_clip_mean: H={H} must satisfy 0 <= H < n={n}")
    if P == 0:
        return out
    L.check(L.lib().rcmarl_clip_mean(vals.data_ptr(), n, P, vals.stride(0), int(H), out.data_ptr(), _stream()),
            "rcmarl_clip_mean")
    return out


def value_job(out, terms, add=None, add_stride=1, add_off=0, add_scale=1.0, n_out=1, softmax=0):
    """terms: list of (weights_tensor, kind, scale)."""
    j = L.ValueJob()
    for t, (w, kind, scale) in enumerate(terms):
        j.w[t] = w.data_ptr()
        j.kind[t] = kind
        j.scale[t] = scale
    j.n_terms = len(terms)
    j.n_out = n_out
    j.softmax = softmax
    j.add = ptr(add)
    j.add_stride = add_stride
    j.add_off = add_off
    j.add_scale = add_scale
    j.out = out.data_ptr()
    j._keep = (out, terms, add)
    return j


def job_array(cls, jobs):
    """ctypes array of the job structs `jobs` (a list or another array; the structs are copied)."""
    return (cls * len(jobs))(*jobs)


def values(rows, jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.ValueJob, jobs)
    L.check(L.lib().rcmarl_values(C.byref(rows), a, len(a), _stream()), "rcmarl_values")


def grad_job(w, target, sums, kind, action_agent=0, target_stride=1, time_idx=None):
    j = L.GradJob()
    j.w, j.target, j.sums, j.kind, j.action_agent = w.data_ptr(), target.data_ptr(), sums.data_ptr(), kind, action_agent
    j.target_stride = target_stride
    j.time_idx = ptr(time_idx)
    j._keep = (w, target, sums, time_idx)
    return j


def grad(rows, jobs, loss_mode, ws=None):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.GradJob, jobs)
    if ws is None:
        ws = workspace()
    L.check(L.lib().rcmarl_grad(C.byref(rows), a, len(a), loss_mode, ws.data_ptr(), ws.numel(), _stream()),
            "rcmarl_grad")


def sgd_job(dst, src, sums, n, coef, first=0, loss_out=None, loss_coef=0.0, loss_accumulate=0):
    j = L.SgdJob()
    j.dst, j.src, j.sums, j.loss_out = dst.data_ptr(), src.data_ptr(), sums.data_ptr(), ptr(loss_out)
    j.n, j.first, j.coef, j.loss_coef, j.loss_accumulate = n, first, coef, loss_coef, loss_accumulate
    j._keep = (dst, src, sums, loss_out)
    return j


def sgd_apply(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.SgdJob, jobs)
    L.check(L.lib().rcmarl_sgd_apply(a, len(a), _stream()), "rcmarl_sgd_apply")


class MinibatchCells:
    """Scratch of the persistent mini-batch kernel (rcmarl_minibatch_fit): zero-initialised {value, sequence} cells plus
    the host-side sequence counter (every step of every call consumes one number, never reused)."""

    def __init__(self, n_jobs=L.MAX_JOBS, max_params=None, device=None):
        if max_params is None:
            max_params = L.param_count(48, 1)
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        self.buf = torch.zeros(L.lib().rcmarl_minibatch_cells_bytes(n_jobs, max_params), dtype=torch.uint8, device=dev)
        self.seq = 1


def minibatch_fit(rows, gjobs, sjobs, epochs, n_times, mb_times, lr, cells):
    """Whole mini-batch fit (all epochs, all steps, all chains) as ONE persistent kernel (csrc/minibatch_persist.cuh)."""
    ga = gjobs if isinstance(gjobs, C.Array) else job_array(L.GradJob, gjobs)
    sa = sjobs if isinstance(sjobs, C.Array) else job_array(L.SgdJob, sjobs)
    steps = L.lib().rcmarl_minibatch_steps(epochs, n_times, mb_times)
    if cells.seq + steps >= 0xFFFF0000:                       # 32-bit sequence numbers: start over on clean cells
        cells.buf.zero_()
        cells.seq = 1
    L.check(L.lib().rcmarl_minibatch_fit(C.byref(rows), ga, sa, len(ga), epochs, n_times, mb_times, lr,
                                         cells.buf.data_ptr(), cells.buf.numel(), cells.seq, _stream()),
            "rcmarl_minibatch_fit")
    cells.seq += steps


def _fit_steps(rows, gjobs, ajobs, epochs, n_times, mb_times):
    """The steps of a Keras fit(batch_size=mb_times rows, shuffle=True) over the grad jobs' permutation tables
    (time_idx of job j: int32 [epochs][n_times] time rows; a mini-batch is those rows x rows.n_envs environments).
    Before each step it points rows and every grad job at the step's rows and does the Keras loss bookkeeping on the
    apply jobs ajobs; it yields the step's row count."""
    tables = [g.time_idx for g in gjobs]
    for e in range(epochs):
        for b in range(0, n_times, mb_times):
            rows.n_rows = min(mb_times, n_times - b) * rows.n_envs
            for g, table in zip(gjobs, tables):
                g.time_idx = table + 4 * (e * n_times + b)
            for a in ajobs:
                if b > 0:
                    a.loss_accumulate = 1                   # the loss is summed over the steps of epoch 0 ...
                if e == 1 and b == 0:
                    a.loss_out = None                       # ... only (history['loss'][0])
            yield rows.n_rows


def minibatch_steps(rows, gjobs, sjobs, epochs, n_times, mb_times, lrs, world=1, allreduce=None, ws=None):
    """The fit of minibatch_fit (same job tables; lrs[j] = learning rate of chain j) as rcmarl_grad -> allreduce() ->
    rcmarl_sgd_apply per step: the data-parallel path without a peer-memory exchange, where allreduce() sums the
    chains' gradient sums over the `world` ranks in place."""
    ga, sa = job_array(L.GradJob, gjobs), job_array(L.SgdJob, sjobs)     # copies: the loop rewrites them
    for n_rows in _fit_steps(rows, ga, sa, epochs, n_times, mb_times):
        for s, lr in zip(sa, lrs):
            s.coef = lr * 2.0 / (n_rows * world)
        grad(rows, ga, L.LOSS_MSE, ws)
        if allreduce is not None:
            allreduce()
        sgd_apply(sa)


def adam_minibatch_steps(rows, gjobs, ajobs, n_times, mb_times, lrs, ts, world=1, allreduce=None, ws=None):
    """One epoch of actor.fit(batch_size=mb_times) with Keras Adam as rcmarl_grad (CE) -> allreduce() ->
    rcmarl_adam_apply per step.  The time_idx of grad job j is a one-epoch permutation table [n_times]; lrs[j] is chain
    j's learning rate and ts[j] the Adam steps it took before.  Returns the number of steps taken (the caller advances
    its step counters by it)."""
    ga, aa = job_array(L.GradJob, gjobs), job_array(L.AdamJob, ajobs)     # copies: the loop rewrites them
    k = 0
    for n_rows in _fit_steps(rows, ga, aa, 1, n_times, mb_times):
        k += 1
        for a, lr, t in zip(aa, lrs, ts):
            a.grad_scale = 1.0 / (n_rows * world)
            a.lr_t = keras_adam_lr_t(lr, t + k)
        grad(rows, ga, L.LOSS_CE, ws)
        if allreduce is not None:
            allreduce()
        adam_apply(aa)
    return k


def adam_job(theta, m, v, sums, n, grad_scale, lr_t, beta1=0.9, beta2=0.999, eps=1e-7, loss_out=None, loss_coef=0.0,
             loss_accumulate=0):
    j = L.AdamJob()
    j.theta, j.m, j.v, j.sums, j.loss_out = theta.data_ptr(), m.data_ptr(), v.data_ptr(), sums.data_ptr(), ptr(loss_out)
    j.n, j.grad_scale, j.lr_t, j.beta1, j.beta2, j.eps, j.loss_coef = n, grad_scale, lr_t, beta1, beta2, eps, loss_coef
    j.loss_accumulate = loss_accumulate
    j._keep = (theta, m, v, sums, loss_out)
    return j


def adam_apply(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.AdamJob, jobs)
    L.check(L.lib().rcmarl_adam_apply(a, len(a), _stream()), "rcmarl_adam_apply")


def keras_adam_lr_t(lr, t, beta1=0.9, beta2=0.999):
    """lr_t of TF-2 Keras Adam at step t >= 1 (SURVEY Appendix A.5)."""
    return float(np.float32(lr * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)))


def team_job(w, kind, msgs=None, msg_stride=0, in_nodes=(), H=0, sums=None, agg_out=None, agg_in=None, rule="clip"):
    """rule: aggregation rule name or rcmarl_agg_rule id (include/rcmarl.h)."""
    j = L.TeamJob()
    j.w, j.msgs, j.msg_stride = w.data_ptr(), ptr(msgs), msg_stride
    j.sums, j.agg_out, j.agg_in = ptr(sums), ptr(agg_out), ptr(agg_in)
    j.kind, j.n_in, j.H, j.rule = kind, len(in_nodes), H, L.agg_rule(rule)
    for k, v in enumerate(in_nodes):
        j.in_nodes[k] = v
    j._keep = (w, msgs, sums, agg_out, agg_in)
    return j


def team(rows, jobs, ws=None):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.TeamJob, jobs)
    if ws is None:
        ws = workspace()
    L.check(L.lib().rcmarl_team(C.byref(rows), a, len(a), ws.data_ptr(), ws.numel(), _stream()), "rcmarl_team")


def consensus_job(dst, msgs, msg_stride, n_hidden, in_nodes, H, rule="clip"):
    """rule: aggregation rule name or rcmarl_agg_rule id (include/rcmarl.h)."""
    j = L.ConsensusJob()
    j.dst, j.msgs, j.msg_stride, j.n_hidden, j.n_in, j.H = dst.data_ptr(), msgs.data_ptr(), msg_stride, n_hidden, len(in_nodes), H
    j.rule = L.agg_rule(rule)
    for k, v in enumerate(in_nodes):
        j.in_nodes[k] = v
    j._keep = (dst, msgs)
    return j


def consensus_hidden(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.ConsensusJob, jobs)
    L.check(L.lib().rcmarl_consensus_hidden(a, len(a), _stream()), "rcmarl_consensus_hidden")


def attack_job(dst, msgs, msg_stride, n, honest, kind, param, seed=0, attacker=0, receiver=0, round=0, epoch=0):
    """kind: attack name ("alie", "ipm", "gauss") or rcmarl_attack_kind id; honest: the message rows of the honest set
    in list order (include/rcmarl.h).  Names are checked here, ids and parameters by the library."""
    j = L.AttackJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.n_honest = len(honest)
    for k, v in enumerate(honest[:L.MAX_NEIGHBOURS]):
        j.honest[k] = v
    if isinstance(kind, str):
        if kind not in L.ATTACKS:
            raise L.RcmarlError(f"unknown attack {kind!r}: expected one of {sorted(L.ATTACKS)}")
        kind = L.ATTACKS[kind]
    j.kind, j.param = int(kind), param
    j.seed, j.attacker, j.receiver, j.round, j.epoch = int(seed), attacker, receiver, round, epoch
    j._keep = (dst, msgs)
    return j


def attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.AttackJob, jobs)
    L.check(L.lib().rcmarl_attack(a, len(a), _stream()), "rcmarl_attack")


def adaptive_attack_job(dst, msgs, msg_stride, n, honest, attack, scale, gamma_out=None):
    """attack: min-max / min-sum attack name ("minmax_uv", ..., "minsum_sgn") or a (rcmarl_adaptive_kind,
    rcmarl_adaptive_dev) pair of ids (include/rcmarl.h); scale: s >= 0.  Names are checked here, ids and limits by the
    library."""
    j = L.AdaptiveAttackJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.gamma_out = ptr(gamma_out)
    j.n_honest = len(honest)
    for k, v in enumerate(honest[:L.MAX_NEIGHBOURS]):
        j.honest[k] = v
    if isinstance(attack, str):
        if not L.is_adaptive_attack(attack):
            raise L.RcmarlError(f"unknown adaptive attack {attack!r}: expected one of {sorted(L.ADAPTIVE_ATTACKS)}")
        attack = L.ADAPTIVE_ATTACKS[attack]
    j.kind, j.dev = int(attack[0]), int(attack[1])
    j.scale = scale
    j._keep = (dst, msgs, gamma_out)
    return j


def adaptive_attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.AdaptiveAttackJob, jobs)
    L.check(L.lib().rcmarl_adaptive_attack(a, len(a), _stream()), "rcmarl_adaptive_attack")


def tailored_attack_job(dst, msgs, msg_stride, n, slots, honest, rule, H, attack, scale, gamma_out=None):
    """slots: the receiver's slot list (in_nodes order, own first), a message row or -1 for a crafted slot; honest: the
    slot indices of the honest set; rule: the receiver's rule name (coordinate-wise "clip", "trim", "wmsr" or
    distance-based "krum", "mkrum", "scclip", "gmed") or a (rcmarl_tailored_family, rule id) pair; attack: "tailored_uv",
    "tailored_std", "tailored_sgn" or an rcmarl_adaptive_dev id; scale: the range multiplier s >= 0.  Names are checked
    here, ids and limits by the library."""
    j = L.TailoredAttackJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.gamma_out = ptr(gamma_out)
    j.n_in = len(slots)
    for k, v in enumerate(slots[:L.MAX_NEIGHBOURS]):
        j.slots[k] = v
    bad = [k for k in honest if not (isinstance(k, (int, np.integer)) and 0 <= k < len(slots))]
    if bad:
        raise L.RcmarlError(f"honest slot indices {bad} are outside the slot list of {len(slots)}")
    j.honest_mask = sum(1 << int(k) for k in set(honest))
    if isinstance(rule, str):
        fam = L.TAILOR_VECTOR if L.is_vector_rule(rule) else L.TAILOR_COORD
        rule = (fam, L.VECTOR_RULES[rule] if fam == L.TAILOR_VECTOR else L.agg_rule(rule))
    j.family, j.rule, j.H = int(rule[0]), int(rule[1]), H
    if isinstance(attack, str):
        if not L.is_tailored_attack(attack):
            raise L.RcmarlError(f"unknown tailored attack {attack!r}: expected one of {sorted(L.TAILORED_ATTACKS)}")
        attack = L.TAILORED_ATTACKS[attack]
    j.dev = int(attack)
    j.scale = scale
    j._keep = (dst, msgs, gamma_out)
    return j


def tailored_attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.TailoredAttackJob, jobs)
    L.check(L.lib().rcmarl_tailored_attack(a, len(a), _stream()), "rcmarl_tailored_attack")


def pipeline_attack_job(dst, msgs, msg_stride, n, slots, honest, rule, H, attack, scale, mixing=None, n_perms=1, seed=0,
                        attacker=0, receiver=0, net=0, round=0, epoch=0, gamma_out=None, model_out=None):
    """rcmarl_pipeline_attack_job: slots, honest, H and scale as tailored_attack_job; rule: the receiver's rule name
    (those of tailored_attack_job, or "dnc") or a (rcmarl_tailored_family, rule id) pair; attack: "pipeline_uv",
    "pipeline_std", "pipeline_sgn", an ARC attack's name ("arc_uv", "arc_std", "arc_sgn": the same job for
    pipeline_arc_attack), a subset attack's name ("subset_uv", "subset_std", "subset_sgn": with rule "mda" or "smea"
    the job for subset_pipeline_attack, else the same job as the ARC attack's), an IOS attack's name ("ios_uv",
    "ios_std", "ios_sgn": with rule "ios" the job for ios_pipeline_attack, else the same job as the subset attack's)
    or an rcmarl_adaptive_dev id; mixing: the receiver's mixing entry (None, "nnm", "bucket" or ("bucket", s), see
    _lib.mixing_entry); n_perms: the attacker's shuffle samples under bucketing; (seed,
    attacker, receiver, net, round, epoch): the Philox key and counter words of those samples; model_out [n]: R_0 of the
    pick.  Names are checked here, ids and limits by the library."""
    if isinstance(attack, str):
        if not (L.is_pipeline_attack(attack) or L.is_arc_attack(attack) or L.is_subset_attack(attack)
                or L.is_ios_attack(attack)):
            names = sorted(L.PIPELINE_ATTACKS) + sorted(L.ARC_ATTACKS) + sorted(L.SUBSET_ATTACKS) + sorted(L.IOS_ATTACKS)
            raise L.RcmarlError(f"unknown pipeline attack {attack!r}: expected one of {names}")
        rule = _chain_family(attack, rule)
        attack = {**L.PIPELINE_ATTACKS, **L.ARC_ATTACKS, **L.SUBSET_ATTACKS, **L.IOS_ATTACKS}[attack]
    if L.is_spectral_rule(rule):
        rule = (L.TAILOR_SPECTRAL, L.SPECTRAL_RULES[rule])
    mixing = L.mixing_entry(mixing)
    j = L.PipelineAttackJob()
    j.attack = tailored_attack_job(dst, msgs, msg_stride, n, slots, honest, rule, H, int(attack), scale, gamma_out)
    j.model_out = ptr(model_out)
    j.mixing = L.PIPE_NONE if mixing is None else L.PIPE_NNM if mixing == "nnm" else L.PIPE_BUCKET
    j.s = mixing[1] if L.is_bucket_mixing(mixing) else 0
    j.n_perms = n_perms
    j.seed, j.attacker, j.receiver, j.net, j.round, j.epoch = int(seed), attacker, receiver, net, round, epoch
    j._keep = (dst, msgs, gamma_out, model_out)
    return j


def _chain_family(attack, rule):
    """(TAILOR_SUBSET, rule id) for a subset or IOS attack's name against "mda" / "smea", (TAILOR_FILTER, FILTER_IOS)
    for an IOS attack's name against "ios", else rule unchanged."""
    if (L.is_subset_attack(attack) or L.is_ios_attack(attack)) and L.is_subset_rule(rule):
        return L.TAILOR_SUBSET, L.SUBSET_RULES[rule]
    if L.is_ios_attack(attack) and L.is_filter_rule(rule):
        return L.TAILOR_FILTER, L.FILTER_RULES[rule]
    return rule


def pipeline_attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.PipelineAttackJob, jobs)
    L.check(L.lib().rcmarl_pipeline_attack(a, len(a), _stream()), "rcmarl_pipeline_attack")


def pipeline_arc_attack(jobs):
    """rcmarl_pipeline_arc_attack: pipeline_attack_job's jobs against receivers that clip (ARC at each job's H)."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.PipelineAttackJob, jobs)
    L.check(L.lib().rcmarl_pipeline_arc_attack(a, len(a), _stream()), "rcmarl_pipeline_arc_attack")


def history_attack_job(dst, msgs, msg_stride, n, slots, honest, rule, H, attack, scale, ref, momentum, momentum_stride,
                       beta, first, own, gamma_out=None, model_out=None):
    """rcmarl_history_attack_job: slots, honest, rule, H and scale as pipeline_attack_job; attack: "history_uv",
    "history_std", "history_sgn", an ARC attack's name (the same job for history_arc_attack), a subset attack's name
    (with rule "mda" or "smea" the job for subset_history_attack, else the same job as the ARC attack's), an IOS
    attack's name (with rule "ios" the job for ios_history_attack, else the same job as the subset attack's) or an
    rcmarl_adaptive_dev id; ref the receiver's reference c [>= n]; momentum its state
    M, row k at momentum + k * momentum_stride (read only); beta in [0, 1); first 1 for the receiver's first step; own:
    the crafted slot indices that receive dst; model_out [n]: R of the pick.  Names and own slots are checked here, ids
    and limits by the library."""
    if isinstance(attack, str):
        if not (L.is_history_attack(attack) or L.is_arc_attack(attack) or L.is_subset_attack(attack)
                or L.is_ios_attack(attack)):
            names = sorted(L.HISTORY_ATTACKS) + sorted(L.ARC_ATTACKS) + sorted(L.SUBSET_ATTACKS) + sorted(L.IOS_ATTACKS)
            raise L.RcmarlError(f"unknown history attack {attack!r}: expected one of {names}")
        rule = _chain_family(attack, rule)
        attack = {**L.HISTORY_ATTACKS, **L.ARC_ATTACKS, **L.SUBSET_ATTACKS, **L.IOS_ATTACKS}[attack]
    if L.is_spectral_rule(rule):
        rule = (L.TAILOR_SPECTRAL, L.SPECTRAL_RULES[rule])
    bad = [k for k in own if not (isinstance(k, (int, np.integer)) and 0 <= k < len(slots))]
    if bad:
        raise L.RcmarlError(f"own slot indices {bad} are outside the slot list of {len(slots)}")
    j = L.HistoryAttackJob()
    j.attack = tailored_attack_job(dst, msgs, msg_stride, n, slots, honest, rule, H, int(attack), scale, gamma_out)
    j.model_out = ptr(model_out)
    j.ref, j.momentum, j.momentum_stride = ref.data_ptr(), momentum.data_ptr(), momentum_stride
    j.beta, j.first = beta, int(first)
    j.own_mask = sum(1 << int(k) for k in set(own))
    j._keep = (dst, msgs, gamma_out, model_out, ref, momentum)
    return j


def history_attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.HistoryAttackJob, jobs)
    L.check(L.lib().rcmarl_history_attack(a, len(a), _stream()), "rcmarl_history_attack")


def subset_pipeline_attack(jobs, arc):
    """rcmarl_subset_pipeline_attack: pipeline_attack_job's jobs against MDA / SMEA receivers (family TAILOR_SUBSET),
    through the receiver's clipping step when arc is true."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.PipelineAttackJob, jobs)
    L.check(L.lib().rcmarl_subset_pipeline_attack(a, len(a), int(arc), _stream()), "rcmarl_subset_pipeline_attack")


def subset_history_attack(jobs, arc):
    """rcmarl_subset_history_attack: history_attack_job's jobs against MDA / SMEA receivers with momentum (family
    TAILOR_SUBSET), through the receiver's clipping step when arc is true."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.HistoryAttackJob, jobs)
    L.check(L.lib().rcmarl_subset_history_attack(a, len(a), int(arc), _stream()), "rcmarl_subset_history_attack")


def ios_pipeline_attack(jobs, arc):
    """rcmarl_ios_pipeline_attack: pipeline_attack_job's jobs against IOS receivers (family TAILOR_FILTER), through the
    receiver's clipping step when arc is true."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.PipelineAttackJob, jobs)
    L.check(L.lib().rcmarl_ios_pipeline_attack(a, len(a), int(arc), _stream()), "rcmarl_ios_pipeline_attack")


def ios_history_attack(jobs, arc):
    """rcmarl_ios_history_attack: history_attack_job's jobs against IOS receivers with momentum (family TAILOR_FILTER),
    through the receiver's clipping step when arc is true."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.HistoryAttackJob, jobs)
    L.check(L.lib().rcmarl_ios_history_attack(a, len(a), int(arc), _stream()), "rcmarl_ios_history_attack")


def history_arc_attack(jobs):
    """rcmarl_history_arc_attack: history_attack_job's jobs against receivers that clip (ARC at each job's H)."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.HistoryAttackJob, jobs)
    L.check(L.lib().rcmarl_history_arc_attack(a, len(a), _stream()), "rcmarl_history_arc_attack")


def dissensus_attack_job(dst, msgs, msg_stride, n, own, honest, n_byz, eps):
    """own: the receiver's message row; honest: the message rows of its honest set in list order; n_byz: the dissensus
    entries of its in_nodes (repeats included); eps >= 0 (include/rcmarl.h).  Limits are checked by the library."""
    j = L.DissensusJob()
    j.dst, j.msgs, j.msg_stride, j.n, j.own = dst.data_ptr(), msgs.data_ptr(), msg_stride, n, own
    j.n_honest = len(honest)
    for k, v in enumerate(honest[:L.MAX_NEIGHBOURS]):
        j.honest[k] = v
    j.n_byz, j.eps = n_byz, eps
    j._keep = (dst, msgs)
    return j


def dissensus_attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.DissensusJob, jobs)
    L.check(L.lib().rcmarl_dissensus_attack(a, len(a), _stream()), "rcmarl_dissensus_attack")


def mimic_attack_job(dst, msgs, msg_stride, n, honest, candidates, z, update, target_out=None):
    """honest: the message rows of the receiver's honest set in list order; candidates: the indices into `honest` that
    may be copied; z: the job's direction state [>= n] float32 (zero: not yet initialised); update: 1 to take a power
    step (include/rcmarl.h).  The indices are checked here, limits by the library."""
    j = L.MimicJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.z, j.target_out = z.data_ptr(), ptr(target_out)
    j.n_honest = len(honest)
    for k, v in enumerate(honest[:L.MAX_NEIGHBOURS]):
        j.honest[k] = v
    bad = [k for k in candidates if not (isinstance(k, (int, np.integer)) and 0 <= k < min(len(honest), 32))]
    if bad:
        raise L.RcmarlError(f"candidate indices {bad} are outside the honest set of {len(honest)}")
    j.candidate_mask = sum(1 << int(k) for k in set(candidates))
    j.update = int(update)
    j._keep = (dst, msgs, z, target_out)
    return j


def mimic_attack(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.MimicJob, jobs)
    L.check(L.lib().rcmarl_mimic_attack(a, len(a), _stream()), "rcmarl_mimic_attack")


def vector_job(dst, msgs, msg_stride, n, in_nodes, H, rule, weights_out=None):
    """rule: distance-based rule name ("krum", "mkrum", "scclip", "gmed") or rcmarl_vector_rule id (include/rcmarl.h).
    Names are checked here, ids and limits by the library."""
    j = L.VectorJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.weights_out = ptr(weights_out)
    j.n_in, j.H = len(in_nodes), H
    for k, v in enumerate(in_nodes[:L.MAX_NEIGHBOURS]):
        j.in_nodes[k] = v
    if isinstance(rule, str):
        if not L.is_vector_rule(rule):
            raise L.RcmarlError(f"unknown distance-based aggregation rule {rule!r}: expected one of {sorted(L.VECTOR_RULES)}")
        rule = L.VECTOR_RULES[rule]
    j.rule = int(rule)
    j._keep = (dst, msgs, weights_out)
    return j


def vector_aggregate(jobs):
    a = jobs if isinstance(jobs, C.Array) else job_array(L.VectorJob, jobs)
    L.check(L.lib().rcmarl_vector_aggregate(a, len(a), _stream()), "rcmarl_vector_aggregate")


def dnc_aggregate(jobs):
    """rcmarl_dnc_aggregate over rcmarl_vector_job jobs (vector_job(..., rule=L.SPECTRAL_DNC, ...))."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.VectorJob, jobs)
    L.check(L.lib().rcmarl_dnc_aggregate(a, len(a), _stream()), "rcmarl_dnc_aggregate")


def subset_aggregate(jobs):
    """rcmarl_subset_aggregate over rcmarl_vector_job jobs (vector_job(..., rule=L.SUBSET_MDA or L.SUBSET_SMEA, ...))."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.VectorJob, jobs)
    L.check(L.lib().rcmarl_subset_aggregate(a, len(a), _stream()), "rcmarl_subset_aggregate")


def ios_aggregate(jobs):
    """rcmarl_ios_aggregate over rcmarl_vector_job jobs (vector_job(..., rule=L.FILTER_IOS, ...))."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.VectorJob, jobs)
    L.check(L.lib().rcmarl_ios_aggregate(a, len(a), _stream()), "rcmarl_ios_aggregate")


def nnm_mix(jobs):
    """rcmarl_nnm_mix over rcmarl_vector_job jobs (vector_job(dst, ..., rule=L.MIX_NNM, weights_out=[n_in * n_in])):
    mixed row k goes to dst + k * msg_stride."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.VectorJob, jobs)
    L.check(L.lib().rcmarl_nnm_mix(a, len(a), _stream()), "rcmarl_nnm_mix")


def arc_clip(jobs):
    """rcmarl_arc_clip over rcmarl_vector_job jobs (vector_job(dst, ..., rule=L.MIX_ARC, weights_out=[n_in])): clipped
    row k goes to dst + k * msg_stride, the factors c to weights_out."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.VectorJob, jobs)
    L.check(L.lib().rcmarl_arc_clip(a, len(a), _stream()), "rcmarl_arc_clip")


def momentum_job(dst, msgs, msg_stride, n, in_nodes, ref, momentum, momentum_stride, beta, first):
    """rcmarl_momentum_job: in_nodes the receiver's message rows (own first); ref the reference c [>= n]; momentum the
    state M, row k at momentum + k * momentum_stride; beta in [0, 1); first 1 for the slots' first step
    (include/rcmarl.h).  Limits are checked by the library."""
    j = L.MomentumJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.ref, j.momentum, j.momentum_stride = ref.data_ptr(), momentum.data_ptr(), momentum_stride
    j.n_in = len(in_nodes)
    for k, v in enumerate(in_nodes[:L.MAX_NEIGHBOURS]):
        j.in_nodes[k] = v
    j.beta, j.first = beta, int(first)
    j._keep = (dst, msgs, ref, momentum)
    return j


def momentum_mix(jobs):
    """rcmarl_momentum_mix over momentum_job jobs: row k of the n_in output rows goes to dst + k * msg_stride, and M
    is updated in place."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.MomentumJob, jobs)
    L.check(L.lib().rcmarl_momentum_mix(a, len(a), _stream()), "rcmarl_momentum_mix")


def reward_mix(r, agents, out=None, scale=1.0):
    """r: [rows, n_agents]; out[row] = scale * sum_k r[row, agents[k]] / len(agents) in list order."""
    n_rows, n_agents = r.shape
    if out is None:
        out = torch.empty(n_rows, dtype=torch.float32, device=r.device)
    arr = (C.c_int32 * len(agents))(*agents)
    L.check(L.lib().rcmarl_reward_mix(r.data_ptr(), n_rows, n_agents, arr, len(agents), scale, out.data_ptr(), _stream()),
            "rcmarl_reward_mix")
    return out


def state_tables(nrow, ncol, scaling=True):
    """(i - mean) / std per coordinate in float64, rounded to float32 (grid_world.py:30-35,70); mean / std are taken over
    the axis' own range, but both tables cover max(nrow, ncol) positions because the reference clips BOTH coordinates
    with nrow - 1 (grid_world.py:55), so y can leave [0, ncol) when nrow > ncol.  scaling=False: identity (the
    reference's Grid_World default)."""
    n = max(nrow, ncol)
    idx = np.arange(n)
    if not scaling:
        t = idx.astype(np.float32)
        return t, t.copy()
    x, y = np.arange(nrow), np.arange(ncol)
    tx = ((idx - np.mean(x)) / np.std(x)).astype(np.float32)
    ty = ((idx - np.mean(y)) / np.std(y)).astype(np.float32)
    return tx, ty


def rollout(actor_w, critic_w, desired, sa, ns, r, time_begin, est, ret, *, n_envs, n_agents, n_episodes, max_ep_len,
            nrow, ncol, gamma, mu=0.1, seed=0, env_offset=0, episode_offset=0, uniforms=None, init_state=None,
            scaling=True, n_active=None):
    A = L.RolloutArgs()
    A.actor_w, A.critic_w, A.desired = actor_w.data_ptr(), critic_w.data_ptr(), desired.data_ptr()
    A.sa, A.ns, A.r = sa.data_ptr(), ns.data_ptr(), r.data_ptr()
    A.time_begin = int(time_begin)
    A.est, A.ret = est.data_ptr(), ret.data_ptr()
    A.uniforms, A.init_state = ptr(uniforms), ptr(init_state)
    A.seed, A.env_offset, A.episode_offset = int(seed), int(env_offset), int(episode_offset)
    A.n_envs, A.n_agents, A.n_episodes, A.max_ep_len = n_envs, n_agents, n_episodes, max_ep_len
    A.nrow, A.ncol, A.gamma, A.mu = nrow, ncol, gamma, mu
    A.n_active = n_agents if n_active is None else int(n_active)
    if max(nrow, ncol) > L.MAX_GRID:
        raise L.RcmarlError(f"grid {nrow}x{ncol} exceeds RCMARL_MAX_GRID = {L.MAX_GRID}")
    tx, ty = state_tables(nrow, ncol, scaling)
    for i in range(len(tx)):
        A.state_tab_x[i] = float(tx[i])
        A.state_tab_y[i] = float(ty[i])
    L.check(L.lib().rcmarl_rollout(C.byref(A), _stream()), "rcmarl_rollout")


def episode_means(x, out=None):
    """x: [n_episodes, n_envs, n_agents] float32 CUDA -> [n_episodes, n_agents] means over the environments."""
    n_ep, n_envs, n_agents = x.shape
    if out is None:
        out = torch.empty(n_ep, n_agents, dtype=torch.float32, device=x.device)
    L.check(L.lib().rcmarl_episode_means(x.data_ptr(), n_ep, n_envs, n_agents, out.data_ptr(), _stream()), "rcmarl_episode_means")
    return out


def env_step(state, action, desired, nrow, reward=None):
    n_envs, n_agents = state.shape[0], state.shape[1]
    if reward is None:
        reward = torch.empty(n_envs, n_agents, dtype=torch.float32, device=state.device)
    L.check(L.lib().rcmarl_env_step(state.data_ptr(), action.data_ptr(), desired.data_ptr(), n_envs, n_agents, nrow,
                                    reward.data_ptr(), _stream()), "rcmarl_env_step")
    return reward


def bucket_job(dst, msgs, msg_stride, n, in_nodes, s, seed=0, receiver=0, net=0, round=0, epoch=0, weights_out=None):
    """rcmarl_bucket_job: in_nodes the receiver's message rows (own first); s the bucket size; (seed, receiver, net,
    round, epoch) the Philox key and counter words of the permutation; weights_out [n_out * n_in] for M
    (include/rcmarl.h).  Limits are checked by the library."""
    j = L.BucketJob()
    j.dst, j.msgs, j.msg_stride, j.n = dst.data_ptr(), msgs.data_ptr(), msg_stride, n
    j.weights_out = ptr(weights_out)
    j.n_in, j.s = len(in_nodes), s
    for k, v in enumerate(in_nodes[:L.MAX_NEIGHBOURS]):
        j.in_nodes[k] = v
    j.seed, j.receiver, j.net, j.round, j.epoch = int(seed), receiver, net, round, epoch
    j._keep = (dst, msgs, weights_out)
    return j


def bucket_mix(jobs):
    """rcmarl_bucket_mix over bucket_job jobs: row r of the n_out = 1 + ceil((n_in - 1) / s) output rows goes to
    dst + r * msg_stride."""
    a = jobs if isinstance(jobs, C.Array) else job_array(L.BucketJob, jobs)
    L.check(L.lib().rcmarl_bucket_mix(a, len(a), _stream()), "rcmarl_bucket_mix")
