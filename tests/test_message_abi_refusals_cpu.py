"""Each message entry point refuses exactly the job tables that the refusal rules of include/rcmarl.h refuse.

The twelve entry points that aggregate, mix or craft whole messages (rcmarl_vector_aggregate, _dnc_aggregate,
_subset_aggregate, _nnm_mix, _bucket_mix, _momentum_mix, _adaptive_attack, _tailored_attack, _pipeline_attack,
_history_attack, _dissensus_attack and _mimic_attack) check every job table before any CUDA call.  Without a device, a
table that passes every check reaches the CUDA runtime and comes back as RCMARL_ERR_CUDA (-3), and a refused one as
RCMARL_ERR_ARG (-1), so the library's decision can be read on any machine.  The calls run in a child process that sees
no device (CUDA_VISIBLE_DEVICES=""): a table the library accepts then never launches a kernel on its made-up addresses.

The tables are seeded and random: 1-32 jobs, random strides (0 and negative among them), node lists with -1 and repeated
slots, and every pointer taken from an arena that packs regions end to end, some of them then moved onto the start, the
end or one float either side of another region.  Overlaps, touching ranges (end == start, which the library accepts) and
exact coincidences are all common.  `refused` below restates the header's refusal rules for each entry point in plain
Python; it is the reference.  Run as a script (python tests/test_message_abi_refusals_cpu.py SEED TABLES), this file
prints the library's return codes for the tables of SEED as JSON; with RCMARL_LIB pointing at another build, that
compares two builds' refusals table by table.
"""
import json
import math
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "resilient-consensus-based-marl_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from rcmarl import _lib as L  # noqa: E402

ERR_ARG, ERR_CUDA = -1, -3
BASE = 1 << 24                          # the arena's first address: far from 0, so that no range wraps
F = 4                                   # bytes per float

# entry point -> (job struct, staging bound in floats or None)
ENTRIES = {
    "rcmarl_vector_aggregate": (L.VectorJob, L.VECTOR_MAX_FLOATS),
    "rcmarl_dnc_aggregate": (L.VectorJob, L.DNC_MAX_FLOATS),
    "rcmarl_subset_aggregate": (L.VectorJob, L.SUBSET_MAX_FLOATS),
    "rcmarl_nnm_mix": (L.VectorJob, L.NNM_MAX_FLOATS),
    "rcmarl_bucket_mix": (L.BucketJob, None),
    "rcmarl_momentum_mix": (L.MomentumJob, None),
    "rcmarl_adaptive_attack": (L.AdaptiveAttackJob, L.ADAPTIVE_MAX_FLOATS),
    "rcmarl_tailored_attack": (L.TailoredAttackJob, L.TAILORED_MAX_FLOATS),
    "rcmarl_pipeline_attack": (L.PipelineAttackJob, L.PIPELINE_MAX_FLOATS),
    "rcmarl_history_attack": (L.HistoryAttackJob, L.HISTORY_MAX_FLOATS),
    "rcmarl_dissensus_attack": (L.DissensusJob, None),
    "rcmarl_mimic_attack": (L.MimicJob, L.MIMIC_MAX_FLOATS),
}


# ---------------------------------------------------------------------------------------------------------------------
# The reference: the header's refusal rules, one entry point at a time.  A job table is refused when one of its jobs is
# or when its ranges collide: a written range that overlaps another written range or a read range of any job.


def rows(base, count, stride, n):
    """The byte ranges of `count` rows of n floats at base + r * stride floats."""
    return [(base + r * stride * F, base + r * stride * F + n * F) for r in range(count)]


def node_rows(base, nodes, stride, n):
    """The byte ranges of the rows base + k * stride floats, k in nodes, less the crafted slots (-1)."""
    return [(base + k * stride * F, base + k * stride * F + n * F) for k in nodes if k >= 0]


def collide(written, read):
    w = np.array(written, dtype=object).reshape(-1, 2)
    r = np.array(read, dtype=object).reshape(-1, 2)
    ww = (w[:, None, 0] < w[None, :, 1]) & (w[None, :, 0] < w[:, None, 1])
    np.fill_diagonal(ww, False)
    wr = (w[:, None, 0] < r[None, :, 1]) & (r[None, :, 0] < w[:, None, 1])
    return bool(ww.any() or wr.any())


def touch(written, read):
    """True if a written range ends where another range starts, or starts where one ends."""
    starts = {a for a, _ in written + read}
    ends = {b for _, b in written + read}
    return any(b in starts for _, b in written) or any(a in ends for a, _ in written)


def bad_rule(family, rule, H, n_rows):
    """An H or rule the receiver's rule refuses for n_rows messages."""
    if not 0 <= H < n_rows:
        return True
    if family == L.TAILOR_COORD:
        return rule not in (L.AGG_CLIP, L.AGG_TRIM, L.AGG_WMSR) or (rule == L.AGG_TRIM and 2 * H >= n_rows)
    if family == L.TAILOR_VECTOR:
        return rule not in (L.VEC_KRUM, L.VEC_MKRUM, L.VEC_SCCLIP, L.VEC_GMED) or \
            (rule in (L.VEC_KRUM, L.VEC_MKRUM) and n_rows < H + 3)
    if family == L.TAILOR_SPECTRAL:
        return rule != L.SPECTRAL_DNC
    return True


def bad_scale(x):
    return not math.isfinite(x) or x < 0


def bad_beta(beta, first):
    return not math.isfinite(beta) or not 0 <= beta < 1 or first not in (0, 1)


def bad_slots(a):
    """What rcmarl_tailored_attack refuses of a job's slots, direction and scale."""
    if not a.dst or not a.msgs or a.n < 1 or not 1 <= a.n_in <= L.MAX_NEIGHBOURS:
        return True
    slots, mask = list(a.slots[:a.n_in]), a.honest_mask
    if any(s < -1 for s in slots) or mask >> a.n_in or mask == 0 or all(s >= 0 for s in slots):
        return True
    if any(s == -1 and (mask >> k) & 1 for k, s in enumerate(slots)):
        return True
    return a.dev not in (L.DEV_UV, L.DEV_STD, L.DEV_SGN) or bad_scale(a.scale)


def check_job(entry, q, bound):
    """(refused, written ranges, read ranges) of one job."""
    w, r = [], []
    if entry in ("rcmarl_vector_aggregate", "rcmarl_dnc_aggregate", "rcmarl_subset_aggregate", "rcmarl_nnm_mix"):
        if not q.dst or not q.msgs or q.n < 1 or not 1 <= q.n_in <= L.MAX_NEIGHBOURS:
            return True, w, r
        nodes = list(q.in_nodes[:q.n_in])
        if min(nodes) < 0:
            return True, w, r
        if entry == "rcmarl_vector_aggregate":
            bad, staged = bad_rule(L.TAILOR_VECTOR, q.rule, q.H, q.n_in), q.n_in + 1
        elif entry == "rcmarl_dnc_aggregate":
            bad, staged = bad_rule(L.TAILOR_SPECTRAL, q.rule, q.H, q.n_in), q.n_in + 2
        elif entry == "rcmarl_subset_aggregate":
            bad, staged = q.rule not in (L.SUBSET_MDA, L.SUBSET_SMEA) or not 0 <= q.H < q.n_in, q.n_in
        else:
            bad, staged = q.rule != L.MIX_NNM or not 0 <= q.H < q.n_in, q.n_in
        if bad or staged * q.n > bound:
            return True, w, r
        if entry == "rcmarl_nnm_mix":
            w += rows(q.dst, q.n_in, q.msg_stride, q.n)
            if q.weights_out:
                w += rows(q.weights_out, 1, 0, q.n_in * q.n_in)
        else:
            w += rows(q.dst, 1, 0, q.n)
            if q.weights_out:
                w += rows(q.weights_out, 1, 0, q.n_in)
        r += node_rows(q.msgs, nodes, q.msg_stride, q.n)
    elif entry == "rcmarl_bucket_mix":
        if not q.dst or not q.msgs or q.n < 1 or not 1 <= q.n_in <= L.MAX_NEIGHBOURS:
            return True, w, r
        nodes = list(q.in_nodes[:q.n_in])
        if min(nodes) < 0 or q.s < 1 or q.net > 1 or q.receiver > 255:
            return True, w, r
        n_out = 1 + -(-(q.n_in - 1) // q.s)
        w += rows(q.dst, n_out, q.msg_stride, q.n)
        if q.weights_out:
            w += rows(q.weights_out, 1, 0, n_out * q.n_in)
        r += node_rows(q.msgs, nodes, q.msg_stride, q.n)
    elif entry == "rcmarl_momentum_mix":
        if not q.dst or not q.msgs or not q.ref or not q.momentum or q.n < 1 or not 1 <= q.n_in <= L.MAX_NEIGHBOURS:
            return True, w, r
        nodes = list(q.in_nodes[:q.n_in])
        if min(nodes) < 0 or bad_beta(q.beta, q.first):
            return True, w, r
        w += rows(q.dst, q.n_in, q.msg_stride, q.n) + rows(q.momentum, q.n_in, q.momentum_stride, q.n)
        r += node_rows(q.msgs, nodes, q.msg_stride, q.n)        # the ref is checked on its own (see refused)
    elif entry == "rcmarl_adaptive_attack":
        if not q.dst or not q.msgs or q.n < 1 or not 1 <= q.n_honest <= L.MAX_NEIGHBOURS:
            return True, w, r
        honest = list(q.honest[:q.n_honest])
        if min(honest) < 0 or q.kind not in (L.ADAPT_MINMAX, L.ADAPT_MINSUM) or q.dev not in (0, 1, 2):
            return True, w, r
        if bad_scale(q.scale) or (q.n_honest + 2) * q.n > bound:
            return True, w, r
        w += rows(q.dst, 1, 0, q.n) + (rows(q.gamma_out, 1, 0, 1) if q.gamma_out else [])
        r += node_rows(q.msgs, honest, q.msg_stride, q.n)
    elif entry in ("rcmarl_tailored_attack", "rcmarl_pipeline_attack", "rcmarl_history_attack"):
        a = q if entry == "rcmarl_tailored_attack" else q.attack
        if bad_slots(a):
            return True, w, r
        n_real = sum(1 for s in a.slots[:a.n_in] if s >= 0)
        dnc = 2 if a.family == L.TAILOR_SPECTRAL else 0
        if entry == "rcmarl_tailored_attack":
            if a.family == L.TAILOR_SPECTRAL or bad_rule(a.family, a.rule, a.H, a.n_in) or (a.n_in + 3) * a.n > bound:
                return True, w, r
        elif entry == "rcmarl_pipeline_attack":
            if q.mixing == L.PIPE_NONE:
                n_rows, n_mixed = a.n_in, 0
            elif q.mixing == L.PIPE_NNM:
                n_rows, n_mixed = a.n_in, a.n_in
            elif q.mixing == L.PIPE_BUCKET:
                if q.s < 1 or not 1 <= q.n_perms <= L.PIPELINE_MAX_PERMS:
                    return True, w, r
                if q.attacker > 255 or q.receiver > 255 or q.net > 1:
                    return True, w, r
                n_rows = 1 + -(-(a.n_in - 1) // q.s)
                n_mixed = n_rows - 1
            else:
                return True, w, r
            if bad_rule(a.family, a.rule, a.H, n_rows) or (n_real + n_mixed + 4 + dnc) * a.n > bound:
                return True, w, r
        else:
            if bad_rule(a.family, a.rule, a.H, a.n_in) or not q.ref or not q.momentum or bad_beta(q.beta, q.first):
                return True, w, r
            own = q.own_mask
            if own == 0 or own >> a.n_in or any((own >> k) & 1 and s >= 0 for k, s in enumerate(a.slots[:a.n_in])):
                return True, w, r
            if (a.n_in + 4 + dnc) * a.n > bound:
                return True, w, r
            r += rows(q.ref, 1, 0, a.n) + rows(q.momentum, a.n_in, q.momentum_stride, a.n)
        w += rows(a.dst, 1, 0, a.n) + (rows(a.gamma_out, 1, 0, 1) if a.gamma_out else [])
        if entry != "rcmarl_tailored_attack" and q.model_out:
            w += rows(q.model_out, 1, 0, a.n)
        r += node_rows(a.msgs, list(a.slots[:a.n_in]), a.msg_stride, a.n)
    elif entry == "rcmarl_dissensus_attack":
        if not q.dst or not q.msgs or q.n < 1 or not 1 <= q.n_honest <= L.MAX_NEIGHBOURS:
            return True, w, r
        honest = list(q.honest[:q.n_honest])
        if q.own < 0 or min(honest) < 0 or not 1 <= q.n_byz <= L.MAX_NEIGHBOURS or bad_scale(q.eps):
            return True, w, r
        w += rows(q.dst, 1, 0, q.n)
        r += node_rows(q.msgs, [q.own] + honest, q.msg_stride, q.n)
    elif entry == "rcmarl_mimic_attack":
        if not q.dst or not q.msgs or not q.z or q.n < 1 or not 1 <= q.n_honest <= L.MAX_NEIGHBOURS:
            return True, w, r
        honest = list(q.honest[:q.n_honest])
        if min(honest) < 0 or q.candidate_mask == 0 or q.candidate_mask >> q.n_honest or q.update not in (0, 1):
            return True, w, r
        if (q.n_honest + 3) * q.n > bound:
            return True, w, r
        w += rows(q.dst, 1, 0, q.n) + rows(q.z, 1, 0, q.n)
        if q.target_out:
            w.append((q.target_out, q.target_out + 4))           # one int32
        r += node_rows(q.msgs, honest, q.msg_stride, q.n)
    return False, w, r


def refused(entry, jobs):
    """(refused, touching): the header's decision on a job table, and whether one of its written ranges touches another
    range end to start."""
    bound = ENTRIES[entry][1]
    if not 1 <= len(jobs) <= L.MAX_JOBS:
        return True, False
    written, read = [], []
    for q in jobs:
        bad, w, r = check_job(entry, q, bound)
        if bad:
            return True, False
        written += w
        read += r
    if entry == "rcmarl_momentum_mix":
        refs = [(q.ref, q.ref + q.n * F) for q in jobs]
        if any(c0 < r1 and r0 < c1 for c0, c1 in refs for r0, r1 in read):
            return True, False                                  # a ref on an in-node row (two refs may coincide)
        read += refs
    return collide(written, read), touch(written, read)


# ---------------------------------------------------------------------------------------------------------------------
# The tables.


class Arena:
    """Regions packed end to end from BASE (gaps of 0, 1 or 16 floats), and the addresses where they start and end."""

    def __init__(self, rng):
        self.rng, self.top, self.marks = rng, BASE, []

    def rows(self, count, stride, n):
        """The base of `count` rows of n floats, stride floats apart (stride may be 0 or negative)."""
        start = self.top + F * self.rng.choice([0, 0, 0, 1, 16])
        span = ((count - 1) * abs(stride) + max(n, 1)) * F
        self.top = start + span
        base = start + (count - 1) * F * max(-stride, 0)
        self.marks += [start, start + span] + [base + k * stride * F for k in range(count)]
        return base

    def take(self, n):
        return self.rows(1, 0, n)

    def common(self):
        """One region of 16 floats that every call returns (refs that coincide)."""
        if not hasattr(self, "_common"):
            self._common = self.take(16)
        return self._common

    def near(self):
        """An address on or one float either side of a region's start or end."""
        return self.rng.choice(self.marks) + F * self.rng.choice([-1, 0, 0, 1])


def _stride(rng, n):
    return rng.choice([n, n, n, n + 1, n + rng.randint(2, 9), max(n - 1, 1), 0, -n])


def _nodes(rng, count, n_rows):
    return [rng.randrange(n_rows) for _ in range(count)]


def _fill(arr, values):
    for i, v in enumerate(values):
        arr[i] = v


def _slots(rng, n_in, n_rows):
    """A valid slot list and honest mask: at least one crafted slot (-1) and one honest real slot."""
    crafted = set(rng.sample(range(n_in), rng.randint(1, n_in - 1)))
    slots = [-1 if k in crafted else rng.randrange(n_rows) for k in range(n_in)]
    real = [k for k in range(n_in) if slots[k] >= 0]
    honest = rng.sample(real, rng.randint(1, len(real)))
    return slots, sum(1 << k for k in honest), sorted(crafted)


def _rule(rng, family, n_in):
    if family == L.TAILOR_COORD:
        return rng.choice([L.AGG_CLIP, L.AGG_TRIM, L.AGG_WMSR]), rng.randint(0, max(0, (n_in - 1) // 2))
    if family == L.TAILOR_VECTOR:
        return rng.choice([L.VEC_KRUM, L.VEC_MKRUM, L.VEC_SCCLIP, L.VEC_GMED]), rng.randint(0, max(0, n_in - 3))
    return L.SPECTRAL_DNC, rng.randint(0, n_in - 1)


def _tailored(rng, arena, a, n, n_rows_stack, msgs, stride, families):
    a.n_in = rng.randint(2, L.MAX_NEIGHBOURS)
    slots, a.honest_mask, crafted = _slots(rng, a.n_in, n_rows_stack)
    _fill(a.slots, slots)
    a.dst, a.msgs, a.msg_stride, a.n = arena.take(n), msgs, stride, n
    a.gamma_out = arena.take(1) if rng.random() < 0.5 else None
    a.family = rng.choice(families)
    a.rule, a.H = _rule(rng, a.family, a.n_in)
    a.dev, a.scale = rng.randrange(3), rng.choice([0.0, 1.0, 2.5])
    return crafted


def make_job(entry, rng, arena, n, n_rows_stack, msgs, stride):
    Job = ENTRIES[entry][0]
    q = Job()
    if Job is L.VectorJob:
        q.n_in = rng.randint(1, L.MAX_NEIGHBOURS)
        _fill(q.in_nodes, _nodes(rng, q.n_in, n_rows_stack))
        q.msgs, q.msg_stride, q.n = msgs, stride, n
        if entry == "rcmarl_vector_aggregate":
            q.rule, q.H = _rule(rng, L.TAILOR_VECTOR, q.n_in)
        else:
            q.rule = rng.randrange(2) if entry == "rcmarl_subset_aggregate" else 0
            q.H = rng.randint(0, q.n_in - 1)
        nnm = entry == "rcmarl_nnm_mix"
        q.dst = arena.rows(q.n_in, stride, n) if nnm else arena.take(n)
        if rng.random() < 0.5:
            q.weights_out = arena.take(q.n_in * q.n_in if nnm else q.n_in)
    elif Job is L.BucketJob:
        q.n_in = rng.randint(1, L.MAX_NEIGHBOURS)
        _fill(q.in_nodes, _nodes(rng, q.n_in, n_rows_stack))
        q.msgs, q.msg_stride, q.n, q.s = msgs, stride, n, rng.randint(1, q.n_in + 1)
        n_out = 1 + -(-(q.n_in - 1) // q.s)
        q.dst = arena.rows(n_out, stride, n)
        if rng.random() < 0.5:
            q.weights_out = arena.take(n_out * q.n_in)
        q.net, q.receiver = rng.randrange(2), rng.randrange(256)
    elif Job is L.MomentumJob:
        q.n_in = rng.randint(1, L.MAX_NEIGHBOURS)
        _fill(q.in_nodes, _nodes(rng, q.n_in, n_rows_stack))
        q.msgs, q.msg_stride, q.n = msgs, stride, n
        q.dst = arena.rows(q.n_in, stride, n)
        q.momentum_stride = _stride(rng, n)
        q.momentum = arena.rows(q.n_in, q.momentum_stride, n)
        q.ref = arena.take(n) if rng.random() < 0.7 else arena.common()
        q.beta, q.first = rng.choice([0.0, 0.5, 0.9]), rng.randrange(2)
    elif Job is L.AdaptiveAttackJob:
        q.n_honest = rng.randint(1, L.MAX_NEIGHBOURS)
        _fill(q.honest, _nodes(rng, q.n_honest, n_rows_stack))
        q.dst, q.msgs, q.msg_stride, q.n = arena.take(n), msgs, stride, n
        q.gamma_out = arena.take(1) if rng.random() < 0.5 else None
        q.kind, q.dev, q.scale = rng.randrange(2), rng.randrange(3), rng.choice([0.0, 1.0, 2.5])
    elif Job is L.TailoredAttackJob:
        _tailored(rng, arena, q, n, n_rows_stack, msgs, stride, [L.TAILOR_COORD, L.TAILOR_VECTOR])
    elif Job is L.PipelineAttackJob:
        _tailored(rng, arena, q.attack, n, n_rows_stack, msgs, stride, [0, 1, 2])
        q.model_out = arena.take(n) if rng.random() < 0.5 else None
        q.mixing = rng.randrange(3)
        q.s, q.n_perms = rng.randint(1, q.attack.n_in), rng.randint(1, L.PIPELINE_MAX_PERMS)
        q.attacker, q.receiver, q.net = rng.randrange(256), rng.randrange(256), rng.randrange(2)
        if q.mixing == L.PIPE_BUCKET:                             # an H the rule allows on the bucketed rows
            q.attack.H = min(q.attack.H, rng.randint(0, 1))
    elif Job is L.HistoryAttackJob:
        crafted = _tailored(rng, arena, q.attack, n, n_rows_stack, msgs, stride, [0, 1, 2])
        q.model_out = arena.take(n) if rng.random() < 0.5 else None
        q.ref = arena.take(n) if rng.random() < 0.7 else arena.common()
        q.momentum_stride = _stride(rng, n)
        q.momentum = arena.rows(q.attack.n_in, q.momentum_stride, n)
        q.beta, q.first = rng.choice([0.0, 0.5, 0.9]), rng.randrange(2)
        q.own_mask = sum(1 << k for k in rng.sample(crafted, rng.randint(1, len(crafted))))
    elif Job is L.DissensusJob:
        q.n_honest = rng.randint(1, L.MAX_NEIGHBOURS)
        _fill(q.honest, _nodes(rng, q.n_honest, n_rows_stack))
        q.own = rng.randrange(n_rows_stack)
        q.dst, q.msgs, q.msg_stride, q.n = arena.take(n), msgs, stride, n
        q.n_byz, q.eps = rng.randint(1, L.MAX_NEIGHBOURS), rng.choice([0.0, 1.0, 2.0])
    else:
        q.n_honest = rng.randint(1, L.MAX_NEIGHBOURS)
        _fill(q.honest, _nodes(rng, q.n_honest, n_rows_stack))
        q.dst, q.msgs, q.msg_stride, q.n = arena.take(n), msgs, stride, n
        q.z = arena.take(n)
        q.target_out = arena.take(1) if rng.random() < 0.5 else None
        q.candidate_mask = rng.randint(1, (1 << q.n_honest) - 1)
        q.update = rng.randrange(2)
    return q


def _set(q, field, value):
    """Set a field of a job, or of its attack for a pipeline or history job."""
    if not hasattr(type(q), field) and hasattr(q, "attack"):
        q = q.attack
    if field in ("in_nodes", "honest", "slots"):
        getattr(q, field)[value[0]] = value[1]
    else:
        setattr(q, field, value)


POINTERS = {
    L.VectorJob: ["dst", "msgs", "weights_out"], L.BucketJob: ["dst", "msgs", "weights_out"],
    L.MomentumJob: ["dst", "msgs", "ref", "momentum"], L.AdaptiveAttackJob: ["dst", "msgs", "gamma_out"],
    L.TailoredAttackJob: ["dst", "msgs", "gamma_out"], L.PipelineAttackJob: ["dst", "msgs", "gamma_out", "model_out"],
    L.HistoryAttackJob: ["dst", "msgs", "gamma_out", "model_out", "ref", "momentum"],
    L.DissensusJob: ["dst", "msgs"], L.MimicJob: ["dst", "msgs", "z", "target_out"],
}


def _breakage(rng, entry, q, bound):
    """One field set to a value at or just past the edge of what the header allows (some of them still allowed)."""
    Job = type(q)
    a = q.attack if hasattr(q, "attack") else q
    count = "n_honest" if hasattr(a, "n_honest") else "n_in"
    nodes = {"n_honest": "honest", "n_in": "slots" if hasattr(a, "slots") else "in_nodes"}[count]
    n_list = getattr(a, count)
    choices = [("n", 0), ("n", -1), (count, 0), (count, L.MAX_NEIGHBOURS + 1), ("n", 1 << 30),
               (nodes, (rng.randrange(max(n_list, 1)), rng.choice([-1, -2]))), (rng.choice(POINTERS[Job]), None)]
    if bound:
        rows_staged = max(n_list, 1) + rng.randint(0, 6)
        choices += [("n", bound // rows_staged), ("n", bound // rows_staged + 1)]
    if hasattr(a, "H"):
        choices += [("H", -1), ("H", a.n_in), ("H", a.n_in - 1), ("H", (a.n_in + 1) // 2),
                    ("rule", rng.choice([-1, 4]))]
    if hasattr(a, "scale"):
        choices += [("scale", rng.choice([-1.0, float("nan"), float("inf"), 1e38 * 10])), ("dev", rng.choice([-1, 3]))]
    if hasattr(a, "honest_mask"):
        choices += [("honest_mask", 0), ("honest_mask", a.honest_mask | (1 << a.n_in)),
                    ("honest_mask", (1 << a.n_in) - 1), ("family", rng.choice([-1, 2, 3]))]
    if hasattr(q, "beta"):
        choices += [("beta", rng.choice([1.0, -0.0, -1e-9, 1 - 2 ** -25, float("nan"), float("inf")])),
                    ("first", rng.choice([-1, 2]))]
    if hasattr(q, "own_mask"):
        choices += [("own_mask", 0), ("own_mask", q.own_mask | (1 << a.n_in)), ("own_mask", (1 << a.n_in) - 1)]
    if hasattr(q, "mixing"):
        choices += [("mixing", rng.choice([-1, 3])), ("s", 0), ("n_perms", rng.choice([0, 17])),
                    ("attacker", 256), ("receiver", 256), ("net", 2)]
    if Job is L.BucketJob:
        choices += [("s", 0), ("s", -3), ("net", 2), ("receiver", 256)]
    if Job is L.AdaptiveAttackJob:
        choices += [("kind", rng.choice([-1, 2]))]
    if Job is L.DissensusJob:
        choices += [("own", -1), ("n_byz", rng.choice([0, 17])), ("eps", rng.choice([-1.0, float("nan")]))]
    if Job is L.MimicJob:
        choices += [("candidate_mask", 0), ("candidate_mask", 1 << a.n_honest), ("update", rng.choice([-1, 2]))]
    field, value = rng.choice(choices)
    _set(q, field, value)


def make_table(entry, rng):
    arena = Arena(rng)
    n0 = rng.choice([1, 2, 3, 5, 8])
    n_rows_stack = rng.randint(1, 20)
    stride = _stride(rng, n0)
    msgs = arena.rows(n_rows_stack, stride, n0)
    jobs = [make_job(entry, rng, arena, rng.choice([n0, n0, n0, rng.randint(1, max(1, abs(stride)) + 1)]),
                     n_rows_stack, msgs, stride)
            for _ in range(rng.choice([1, 1, 2, 3, 4, 8, rng.randint(1, L.MAX_JOBS), L.MAX_JOBS]))]
    for _ in range(rng.choice([0, 0, 1, 1, 2, 3])):           # move a pointer onto or next to another region
        q = rng.choice(jobs)
        _set(q, rng.choice([f for f in POINTERS[type(q)] if f != "msgs"] + ["msgs"]), arena.near())
    if rng.random() < 0.25:
        _breakage(rng, entry, rng.choice(jobs), ENTRIES[entry][1])
    return jobs


def tables(seed, count):
    """{entry: [job list]} of `count` seeded tables per entry point."""
    out = {}
    for i, entry in enumerate(ENTRIES):
        rng = random.Random(seed * 1000003 + i)
        out[entry] = [make_table(entry, rng) for _ in range(count)]
    return out


def library_codes(seed, count):
    """The library's return code for every table of `seed`, in this process."""
    lib = L.lib()
    codes = {}
    for entry, ts in tables(seed, count).items():
        Job = ENTRIES[entry][0]
        f = getattr(lib, entry)
        codes[entry] = [f((Job * len(jobs))(*jobs), len(jobs), None) for jobs in ts]
    return codes


def _vector_codes(dsts):
    """The library's return codes for one 3-node scclip job of 10-float rows at BASE, at each dst."""
    j = L.VectorJob()
    j.msgs, j.msg_stride, j.n, j.n_in, j.H, j.rule = BASE, 10, 10, 3, 1, L.VEC_SCCLIP
    _fill(j.in_nodes, [0, 1, 2])
    codes = []
    for dst in dsts:
        j.dst = dst
        codes.append(L.lib().rcmarl_vector_aggregate((L.VectorJob * 1)(j), 1, None))
    return codes


def without_a_device(*args):
    """This file run as a script with `args`, in a child process that sees no CUDA device: its JSON output."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, os.path.abspath(__file__), *map(str, args)], env=env,
                         capture_output=True, text=True, timeout=600, check=True)
    return json.loads(out.stdout)


# ---------------------------------------------------------------------------------------------------------------------


def test_every_entry_point_refuses_exactly_what_the_header_refuses():
    seed, count = 20261018, 300
    codes = without_a_device(seed, count)
    for entry, ts in tables(seed, count).items():
        got = codes[entry]
        assert len(got) == len(ts) and set(got) <= {ERR_ARG, ERR_CUDA}, (entry, set(got))
        want = [refused(entry, jobs) for jobs in ts]
        wrong = [i for i, (c, (bad, _)) in enumerate(zip(got, want)) if (c == ERR_ARG) != bad]
        assert not wrong, f"{entry}: tables {wrong[:10]} ({len(wrong)} of {count}) decided unlike the header"
        accepted = sum(1 for c in got if c == ERR_CUDA)
        assert count // 20 <= accepted <= count - count // 20, (entry, accepted)    # both outcomes are common
        assert any(t for bad, t in want if not bad), entry                          # a touching range accepted


def test_a_range_that_ends_where_another_starts_is_accepted():
    """rcmarl_vector_aggregate with one 3-node scclip job: a disjoint dst and a dst that starts exactly where the last
    in-node row ends are accepted (they reach the CUDA runtime); a dst one float earlier is refused."""
    end = BASE + 3 * 10 * F
    assert without_a_device("vector", end + 4096, end, end - F) == [ERR_CUDA, ERR_CUDA, ERR_ARG]


if __name__ == "__main__":
    if sys.argv[1] == "vector":
        print(json.dumps(_vector_codes([int(x) for x in sys.argv[2:]])))
    else:
        print(json.dumps(library_codes(int(sys.argv[1]), int(sys.argv[2]))))
