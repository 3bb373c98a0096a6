"""Batched RPBCAC training engine (device-resident; one process per GPU).

Restates training/train_agents.py:46-163 for N independent environments that
share one set of agents (SURVEY Appendix C): the replay buffer is one
time-major tensor in HBM, the rollout of a whole fixed-policy block is ONE
kernel, and every phase of the update round is a handful of fused launches
over all agents (csrc/, C ABI in include/rcmarl.h).  With n_envs == 1 and
injected randomness it reproduces the reference update for update.

Data-parallel (SURVEY 8e): each rank owns n_envs environments and their buffer
rows for ever; parameters are replicated; the only exchange is one all-reduce
of the packed UNSCALED gradient sums per SGD / Adam / projection step.
"""
import functools
import os

import numpy as np
import torch

from . import _lib as L
from . import dist_util, nets, ops

COOP, GREEDY, MALICIOUS, FAULTY, BYZANTINE = "Cooperative", "Greedy", "Malicious", "Faulty", "Byzantine"
PAD = "(unused agent slot)"


class Trainer:
    def __init__(self, *, labels, in_nodes, weights, desired, n_envs=1, nrow=5, ncol=5, gamma=0.9, H=0,
                 fast_lr=0.01, slow_lr=0.01, max_ep_len=20, n_ep_fixed=50, n_epochs=10, buffer_size=2000,
                 common_reward=False, mu=0.1, seed=0, device=None, rank=0, world=1, group=None,
                 perm_source=None, local_steps=5, mb_epochs=10, mb_times=32, actor_mb_times=200,
                 capacity_times=None, adam_state=None, scaling=True, fixed_initial_state=None, aggregation="clip",
                 attack=None, mixing=None, momentum=None, clipping=None):
        L.lib()
        # Any team size up to 16 (main.py:26): the kernels are instantiated for 5 and 16 agents, a team of n_real agents
        # runs on the next instantiation with the extra agent slots zero (inputs and W1 rows, rcmarl/nets.py) -- exactly the
        # n_real-agent problem.  self.NA is the kernel instantiation, self.n_real the team.
        self.n_real = len(labels)
        try:
            NA = nets.kernel_agents(self.n_real)
        except ValueError as ex:
            raise L.RcmarlError(str(ex))
        self.NA = NA
        self.labels = list(labels) + [PAD] * (NA - self.n_real)
        self.in_nodes = [list(x) for x in in_nodes]
        self.coop = [i for i, l in enumerate(self.labels) if l == COOP]
        self.N, self.nrow, self.ncol = int(n_envs), int(nrow), int(ncol)
        self.gamma, self.mu = float(gamma), float(mu)
        # per-agent trimming parameter H and fast learning rate (agents/resilient_CAC_agents.py:28-36 stores both per agent)
        n_real = self.n_real
        self.H = [int(H)] * n_real if np.isscalar(H) else [int(x) for x in H]
        self.fast_lr = [float(fast_lr)] * n_real if np.isscalar(fast_lr) else [float(x) for x in fast_lr]
        if len(self.H) != n_real or len(self.fast_lr) != n_real:
            raise L.RcmarlError("H / fast_lr must be scalars or one value per agent")
        self.H += [0] * (NA - n_real)
        self.fast_lr += [self.fast_lr[0]] * (NA - n_real)
        # per-agent resilient aggregation rule of the consensus and projection steps ("clip" is the reference's),
        # checked against each cooperative agent's neighbour count and H before anything runs on the device
        agg = [aggregation] * n_real if isinstance(aggregation, (str, int)) else list(aggregation)
        if len(agg) != n_real:
            raise L.RcmarlError("aggregation must be one rule or one rule per agent")
        # A distance-based rule ("krum", "mkrum", "scclip", "gmed") aggregates whole messages into one extra message row
        # per such agent; its consensus and team jobs then read that row as their only in-node under clip, which returns
        # it exactly (the projection target phi.W3 + b3 is linear in the head).
        # The spectral rule "dnc" (divide-and-conquer) does the same through a launch of its own, and so do the exact
        # subset-selection rules "mda" and "smea" (rcmarl_subset_rule), and the iterative outlier scissor "ios"
        # (rcmarl_filter_rule).
        self.vector_rule = [L.VECTOR_RULES[a] if L.is_vector_rule(a) else None for a in agg] + [None] * (NA - n_real)
        self.dnc = [L.is_spectral_rule(a) for a in agg] + [False] * (NA - n_real)
        self.subset_rule = [L.SUBSET_RULES[a] if L.is_subset_rule(a) else None for a in agg] + [None] * (NA - n_real)
        self.ios = [L.is_filter_rule(a) for a in agg] + [False] * (NA - n_real)
        self.aggregation = [L.AGG_CLIP if L.is_vector_rule(a) or L.is_spectral_rule(a) or L.is_subset_rule(a)
                            or L.is_filter_rule(a) else L.agg_rule(a) for a in agg] + [L.AGG_CLIP] * (NA - n_real)

        def check_rule(i, n):
            if self.vector_rule[i] is not None:
                L.check_vector_rule(agg[i], self.H[i], n)
            elif self.dnc[i]:
                L.check_spectral_rule(self.H[i], n)
            elif self.subset_rule[i] is not None:
                L.check_subset_rule(self.H[i], n)
            elif self.ios[i]:
                L.check_filter_rule(self.H[i], n)
            else:
                L.check_aggregation(agg[i], self.H[i], n)
        for i in self.coop:
            check_rule(i, len(self.in_nodes[i]))
        # Pre-aggregation mixing before a cooperative agent's rule, which then reads the mixed rows in place of its
        # received messages with the same H: nearest-neighbour mixing ("nnm", rcmarl_nnm_mix) gives n_in mixed rows;
        # bucketing (("bucket", s), rcmarl_bucket_mix) gives the own row and ceil((n_in - 1) / s) bucket means, so the
        # rule is checked again at that smaller count
        one = mixing is None or isinstance(mixing, str) or L.is_bucket_mixing(mixing)
        mix = [mixing] * n_real if one else list(mixing)
        if len(mix) != n_real:
            raise L.RcmarlError("mixing must be None, one mixing rule or one entry per agent")
        self.mixing = [None] * NA
        for i in range(n_real):
            if mix[i] is None:
                continue
            if i in self.coop:
                n_in = len(self.in_nodes[i])
                L.check_mixing(mix[i], self.H[i], n_in)
                self.mixing[i] = L.mixing_entry(mix[i])
                if L.is_bucket_mixing(self.mixing[i]):
                    n_out = L.mixed_rows(self.mixing[i], n_in)
                    try:
                        check_rule(i, n_out)
                    except L.RcmarlError as ex:
                        raise L.RcmarlError(f"agent {i} buckets its {n_in} messages into {n_out} rows (mixing "
                                            f"{self.mixing[i]!r}): {ex}") from None
            else:                                  # only cooperative agents aggregate: the name alone is checked
                L.check_mixing(mix[i], 0, 1)
        # Per-neighbour momentum (rcmarl_momentum_mix) before a cooperative agent's rule, which then reads n_in momentum
        # rows, one per slot, with the same H: None, one beta for every agent or one entry per agent
        mom = [momentum] * n_real if momentum is None or np.isscalar(momentum) else list(momentum)
        if len(mom) != n_real:
            raise L.RcmarlError("momentum must be None, one beta or one entry per agent")
        self.momentum = [None] * NA
        for i in range(n_real):
            if mom[i] is None:
                continue
            beta = L.check_momentum(mom[i])
            if i not in self.coop:                 # only cooperative agents aggregate: beta alone is checked
                continue
            if self.mixing[i] is not None:
                raise L.RcmarlError(f"agent {i} takes both momentum and mixing {self.mixing[i]!r}: at most one "
                                    "pre-aggregation step per agent")
            self.momentum[i] = beta
        # Adaptive robust clipping (rcmarl_arc_clip) after a cooperative agent's momentum step and before its mixing
        # step and rule, which then read n_in clipped rows with the same H: None, "arc" or one entry per agent
        clip = list(clipping) if isinstance(clipping, (list, tuple)) else [clipping] * n_real
        if len(clip) != n_real:
            raise L.RcmarlError("clipping must be None, 'arc' or one entry per agent")
        self.clipping = [None] * NA
        for i in range(n_real):
            L.check_clipping(clip[i])
            if i in self.coop:                     # only cooperative agents aggregate: the name alone is checked
                self.clipping[i] = clip[i]
        self._init_attacks(attack)
        for e in self.tailor_pairs + self.pipe_pairs + self.hist_pairs + self.arc_pairs + self.subset_pairs:
            b, j, _ = self.byz_pairs[e]            # no rule-aware attack models the iterative outlier scissor
            if self.ios[j]:
                name = ('tailored' if e in self.tailor_pairs else 'pipeline' if e in self.pipe_pairs
                        else 'history' if e in self.hist_pairs else 'ARC' if e in self.arc_pairs else 'subset')
                raise L.RcmarlError(f"Byzantine agent {b} runs a {name} attack against agent {j}, whose rule "
                                    f"{agg[j]!r} the attack does not model")
        for e in self.tailor_pairs + self.pipe_pairs:   # neither attack models the receiver's history
            b, j, _ = self.byz_pairs[e]
            if self.momentum[j] is not None:
                raise L.RcmarlError(f"Byzantine agent {b} runs a {'tailored' if e in self.tailor_pairs else 'pipeline'} "
                                    f"attack against agent {j}, whose momentum the attack does not model")
        for e in self.tailor_pairs + self.pipe_pairs + self.hist_pairs:   # none models the receiver's clipping
            b, j, _ = self.byz_pairs[e]
            if self.clipping[j] is not None:
                name = 'tailored' if e in self.tailor_pairs else 'pipeline' if e in self.pipe_pairs else 'history'
                raise L.RcmarlError(f"Byzantine agent {b} runs a {name} attack against agent {j}, whose clipping "
                                    f"{self.clipping[j]!r} the attack does not model")
        for e in self.tailor_pairs:                # rcmarl_tailored_attack models neither the DnC rule nor mixing
            b, j, _ = self.byz_pairs[e]
            if self.dnc[j]:
                raise L.RcmarlError(f"Byzantine agent {b} runs a tailored attack against agent {j}, whose rule 'dnc' "
                                    "the tailored attack does not model")
            if self.mixing[j] is not None:
                raise L.RcmarlError(f"Byzantine agent {b} runs a tailored attack against agent {j}, whose mixing "
                                    f"{self.mixing[j]!r} the tailored attack does not model")
        for e in self.tailor_pairs + self.pipe_pairs + self.hist_pairs + self.arc_pairs:   # none models mda / smea
            b, j, _ = self.byz_pairs[e]
            if self.subset_rule[j] is not None:
                name = ('tailored' if e in self.tailor_pairs else 'pipeline' if e in self.pipe_pairs
                        else 'history' if e in self.hist_pairs else 'ARC')
                raise L.RcmarlError(f"Byzantine agent {b} runs a {name} attack against agent {j}, whose rule "
                                    f"{agg[j]!r} the attack does not model")
        # an ARC job stages k_clip clipped rows on top of its base job's
        for e in self.arc_pairs + self.subset_pairs + self.ios_pairs:
            b, j, _ = self.byz_pairs[e]
            n_real = sum(k >= 0 for k in self._tailored_slots(j)[0])
            kc = L.arc_count(self.H[j], len(self.in_nodes[j])) if self.clipping[j] is not None else 0
            floats, bound = self._arc_staging(j, n_real, kc)
            if self.subset_rule[j] is not None:    # a subset job stages as its ARC form, under a bound of its own
                bound = L.SUBSET_ATTACK_MAX_FLOATS
            if floats > bound:
                name = 'an ARC' if e in self.arc_pairs else 'a subset' if e in self.subset_pairs else 'an IOS'
                raise L.RcmarlError(f"Byzantine agent {b} runs {name} attack against agent {j}, whose job stages "
                                    f"{floats} floats, more than the {bound} the library admits")
        # row of the aggregate of each cooperative agent with a distance-based rule, after the Byzantine pair rows, then
        # that of each cooperative agent on dnc, then that of each on mda / smea, then that of each on ios
        self.vec_agents = [i for i in self.coop if self.vector_rule[i] is not None]
        self.vec_row = {i: NA + len(self.byz_pairs) + q for q, i in enumerate(self.vec_agents)}
        self.dnc_agents = [i for i in self.coop if self.dnc[i]]
        self.dnc_row = {i: NA + len(self.byz_pairs) + len(self.vec_agents) + q for q, i in enumerate(self.dnc_agents)}
        self.subset_agents = [i for i in self.coop if self.subset_rule[i] is not None]
        self.subset_row = {i: NA + len(self.byz_pairs) + len(self.vec_agents) + len(self.dnc_agents) + q
                           for q, i in enumerate(self.subset_agents)}
        self.ios_agents = [i for i in self.coop if self.ios[i]]
        self.ios_row = {i: NA + len(self.byz_pairs) + len(self.vec_agents) + len(self.dnc_agents)
                        + len(self.subset_agents) + q for q, i in enumerate(self.ios_agents)}
        # then the mixed rows of each cooperative agent that mixes (n_in for nnm, n_out for bucketing): mixed row k at
        # mix_row[i] + k
        self.mix_agents = [i for i in self.coop if self.mixing[i] is not None]
        self.mix_row, row = {}, NA + len(self.byz_pairs) + len(self.vec_agents) + len(self.dnc_agents) \
            + len(self.subset_agents) + len(self.ios_agents)
        for i in self.mix_agents:
            self.mix_row[i] = row
            row += L.mixed_rows(self.mixing[i], len(self.in_nodes[i]))
        # then the momentum rows of each cooperative agent with momentum: slot k's row at mom_row[i] + k
        self.mom_agents = [i for i in self.coop if self.momentum[i] is not None]
        self.mom_row = {}
        for i in self.mom_agents:
            self.mom_row[i] = row
            row += len(self.in_nodes[i])
        # then the clipped rows of each cooperative agent that clips: slot k's row at arc_row[i] + k
        self.arc_agents = [i for i in self.coop if self.clipping[i] is not None]
        self.arc_row = {}
        for i in self.arc_agents:
            self.arc_row[i] = row
            row += len(self.in_nodes[i])
        self.slow_lr = [float(slow_lr)] * NA if np.isscalar(slow_lr) else [float(x) for x in slow_lr] + [0.0] * (NA - n_real)
        self.max_ep_len, self.n_ep_fixed, self.n_epochs = int(max_ep_len), int(n_ep_fixed), int(n_epochs)
        self.block = self.max_ep_len * self.n_ep_fixed                    # time rows per fixed-policy block
        self.buffer_size = int(buffer_size)                               # in time rows (train_agents.py:158)
        self.common_reward = bool(common_reward)
        self.seed, self.rank, self.world, self.group = int(seed), int(rank), int(world), group
        self.local_steps, self.mb_epochs = int(local_steps), int(mb_epochs)
        self.mb_times, self.actor_mb_times = int(mb_times), int(actor_mb_times)
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.perm_source = perm_source
        self._perm_gen = torch.Generator(device="cpu")
        self._perm_gen.manual_seed(self.seed * 7919 + 17)
        self.episodes_done = 0
        # Grid_World(scaling=..., randomize_state=False, initial_state=...) of the reference (grid_world.py:21-45)
        self.scaling = bool(scaling)
        self.fixed_initial_state = None if fixed_initial_state is None else np.asarray(fixed_initial_state, np.int32).reshape(NA, 2)
        self._fixed_init_dev = None

        self.PA, self.PC, self.PT = L.param_count(2 * NA, 5), L.param_count(2 * NA, 1), L.param_count(3 * NA, 1)
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.actor = torch.zeros(NA, self.PA, **f32)
        self.critic = torch.zeros(NA, self.PC, **f32)
        self.tr = torch.zeros(NA, self.PT, **f32)
        self.critic_local = torch.zeros(NA, self.PC, **f32)
        for i, w in enumerate(weights):
            self.actor[i].copy_(torch.as_tensor(nets.pack_padded(w[0], 2 * NA)))
            self.critic[i].copy_(torch.as_tensor(nets.pack_padded(w[1], 2 * NA)))
            self.tr[i].copy_(torch.as_tensor(nets.pack_padded(w[2], 3 * NA)))
            self.critic_local[i].copy_(torch.as_tensor(nets.pack_padded(w[3] if len(w) > 3 else w[1], 2 * NA)))
        # transmitted messages: row i is agent i's; row NA + e is the message crafted for Byzantine pair e; row
        # vec_row[i] / dnc_row[i] / subset_row[i] / ios_row[i] the aggregate of cooperative agent i's distance-based /
        # dnc / mda or smea / ios rule; mix_row[i] + k its mixed message k; mom_row[i] + k its momentum row of slot k;
        # arc_row[i] + k its clipped row of slot k
        n_rows = NA + len(self.byz_pairs) + len(self.vec_agents) + len(self.dnc_agents) + len(self.subset_agents) \
            + len(self.ios_agents) \
            + sum(L.mixed_rows(self.mixing[i], len(self.in_nodes[i])) for i in self.mix_agents) \
            + sum(len(self.in_nodes[i]) for i in self.mom_agents) + sum(len(self.in_nodes[i]) for i in self.arc_agents)
        self.msg_c = torch.zeros(n_rows, self.PC, **f32)
        self.msg_t = torch.zeros(n_rows, self.PT, **f32)
        # w_k of each distance-based aggregate of the last epoch: row 2q critic, 2q + 1 TR of vec_agents[q]
        self.vec_weights = torch.zeros(2 * len(self.vec_agents), L.MAX_NEIGHBOURS, **f32) if self.vec_agents else None
        # ... and of each dnc aggregate: row 2q critic, 2q + 1 TR of dnc_agents[q]
        self.dnc_weights = torch.zeros(2 * len(self.dnc_agents), L.MAX_NEIGHBOURS, **f32) if self.dnc_agents else None
        # ... and of each mda / smea aggregate: row 2q critic, 2q + 1 TR of subset_agents[q]
        self.subset_weights = (torch.zeros(2 * len(self.subset_agents), L.MAX_NEIGHBOURS, **f32)
                               if self.subset_agents else None)
        # ... and of each ios aggregate: row 2q critic, 2q + 1 TR of ios_agents[q]
        self.ios_weights = torch.zeros(2 * len(self.ios_agents), L.MAX_NEIGHBOURS, **f32) if self.ios_agents else None
        # mixing matrix M (row-major [n_rows][n_in], n_rows = len(_rule_nodes(i))) of each agent that mixes: row 2q
        # critic, 2q + 1 TR of mix_agents[q]
        self.mix_weights = torch.zeros(2 * len(self.mix_agents), L.MAX_NEIGHBOURS ** 2, **f32) if self.mix_agents else None
        # clipping factors c of each agent that clips: row 2q critic, 2q + 1 TR of arc_agents[q]
        self.arc_weights = torch.zeros(2 * len(self.arc_agents), L.MAX_NEIGHBOURS, **f32) if self.arc_agents else None
        # gamma of each adaptive, tailored, pipeline, history, ARC or subset attack of the last epoch: row q =
        # gamma_pairs[q], columns critic, TR
        self.att_gamma = torch.zeros(len(self.gamma_pairs), 2, **f32) if self.gamma_pairs else None
        # the mimic attack's direction state z of each mimic pair (row q = mimic_pairs[q]; [q, 0, :PC] critic, [q, 1] TR),
        # the index into S_j each copied in the last epoch, and the power steps each has taken (host)
        self.mimic_z = torch.zeros(len(self.mimic_pairs), 2, self.PT, **f32) if self.mimic_pairs else None
        self.mimic_target = (torch.zeros(len(self.mimic_pairs), 2, dtype=torch.int32, device=self.dev)
                             if self.mimic_pairs else None)
        self.mimic_steps = [0] * len(self.mimic_pairs)
        # the momentum state M of each agent with momentum (row q = mom_agents[q]; [q, 0, k, :PC] critic slot k, [q, 1]
        # TR), and the momentum steps each has taken (host; its first step ignores M)
        self.momentum_M = (torch.zeros(len(self.mom_agents), 2, L.MAX_NEIGHBOURS, self.PT, **f32)
                           if self.mom_agents else None)
        self.momentum_steps = [0] * len(self.mom_agents)
        self.adam_m = torch.zeros(NA, self.PA, **f32)
        self.adam_v = torch.zeros(NA, self.PA, **f32)
        self.adam_t = [0] * NA
        if adam_state is not None:
            for i, st in enumerate(adam_state):
                if st is not None:
                    self.adam_m[i].copy_(st[0]); self.adam_v[i].copy_(st[1]); self.adam_t[i] = int(st[2])
        des = np.zeros((NA, 2), np.int32)
        des[:self.n_real] = np.asarray(desired, np.int32).reshape(self.n_real, 2)
        self.desired = torch.as_tensor(des).to(self.dev)

        # replay buffer (time-major, row = t * N + e); capacity = buffer_size + one block
        self.Tcap = int(capacity_times) if capacity_times else self.buffer_size + self.block
        rows = self.Tcap * self.N
        self.sa = torch.zeros(rows, 3 * NA, **f32)
        self.ns = torch.zeros(rows, 2 * NA, **f32)
        self.r = torch.zeros(rows, NA, **f32)
        self.t_filled = 0
        # per-row scratch
        self.tdt = torch.zeros(NA, rows, **f32)          # critic TD targets (train_agents.py / res..py:114-115)
        n_mal = sum(l == MALICIOUS for l in self.labels)
        self.tdt_local = torch.zeros(max(n_mal, 1), rows if n_mal else 1, **f32)
        self.delta = torch.zeros(NA, rows, **f32)        # TD errors (actor window), indexed by absolute buffer row
        self.r_coop = torch.zeros(rows, **f32)
        self.neg_r_coop = torch.zeros(rows if n_mal else 1, **f32)
        # reduction outputs (contiguous so that one all-reduce covers a whole launch)
        self.sums_fit = torch.zeros(2 * NA, self.PT + 1, **f32)
        self.sums_mb = torch.zeros(3 * NA, self.PT + 1, **f32)
        self.sums_team = torch.zeros(2 * NA, 22, **f32)
        self.sums_actor = torch.zeros(NA, self.PA + 1, **f32)
        self.loss_c = torch.zeros(NA, **f32)
        self.loss_t = torch.zeros(NA, **f32)
        self.loss_a = torch.zeros(NA, **f32)
        self.ws = ops.workspace(L.MAX_JOBS, self.PT)      # the TR net (3 * NA inputs) is the largest
        # scratch of the persistent mini-batch kernel (rcmarl_minibatch_fit)
        self.mb_cells = ops.MinibatchCells(L.MAX_JOBS, self.PT, self.dev)
        self.launches = 0                                 # kernels launched by this engine (bench: gpu_launches)
        self.profile = None                               # bench.py: {"fit_grad": [(start_evt, end_evt), ...], ...}
        self.h2d_bytes = 4 * sum(x.numel() for x in (self.actor, self.critic, self.tr, self.critic_local))
        self.d2h_bytes = 0
        # data parallel: exchange gradient sums inside the reduction kernels over NVLink peer memory (csrc/comm.cuh);
        # RCMARL_PEER_COMM=0 selects one NCCL all-reduce per step instead
        self.comm = None
        if self.world > 1 and os.environ.get("RCMARL_PEER_COMM", "1") != "0":
            self.comm = self._try_peer_comm()

    # ------------------------------------------------------------------ helpers
    def _init_attacks(self, attack):
        """Check the Byzantine agents' attacks and list the (attacker, cooperative receiver) pairs, each with its own
        crafted message row, before anything runs on the device.  attack: None, one (name, param) for every Byzantine
        agent, or one entry per agent (None for the agents that are not Byzantine)."""
        n_real, lab = self.n_real, self.labels
        if attack is None or (isinstance(attack, tuple) and len(attack) == 2 and isinstance(attack[0], str)):
            att = [attack if lab[i] == BYZANTINE else None for i in range(n_real)]
        else:
            att = list(attack)
            if len(att) != n_real:
                raise L.RcmarlError("attack must be one (name, param) pair or one entry per agent")
        self.attack = [None] * n_real
        for i in range(n_real):
            if (att[i] is None) != (lab[i] != BYZANTINE):
                raise L.RcmarlError(f"agent {i} ({lab[i]}): " + ("a Byzantine agent needs an attack" if att[i] is None
                                                                 else "only a Byzantine agent takes an attack"))
            if att[i] is not None:
                self.attack[i] = L.check_attack(att[i])
        # pair e = (attacker b, receiver j, honest set S_j: the cooperative agents of in_nodes[j] in list order)
        self.byz_pairs = []
        for b in range(n_real):
            if lab[b] != BYZANTINE:
                continue
            for j in self.coop:
                if b in self.in_nodes[j]:
                    honest = [k for k in self.in_nodes[j] if lab[k] == COOP]
                    if not honest:
                        raise L.RcmarlError(f"cooperative agent {j} hears Byzantine agent {b} but no cooperative agent: "
                                            "the attack has no honest set")
                    self.byz_pairs.append((b, j, honest))
        # the pairs whose attacker runs a min-max / min-sum attack (rcmarl_adaptive_attack; check_attack gives its kind
        # as a (kind, dev) pair): their messages are crafted by a launch of their own
        self.adapt_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs) if isinstance(self.attack[b][0], tuple)]
        # the pairs whose attacker runs a rule-aware attack (rcmarl_tailored_attack, kind L.TailoredKind): a launch of
        # their own too, after the adaptive one
        self.tailor_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                             if isinstance(self.attack[b][0], L.TailoredKind)]
        # the pairs whose attacker runs a pipeline-aware attack (rcmarl_pipeline_attack, kind L.PipelineKind), which
        # models the receiver's mixing step and every rule, DnC included: a launch of their own, after the tailored one
        self.pipe_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                           if isinstance(self.attack[b][0], L.PipelineKind)]
        # the pairs whose attacker runs a momentum-aware attack (rcmarl_history_attack, kind L.HistoryKind): against a
        # receiver with momentum a launch of their own, after the pipeline one; against one without, a pipeline job
        self.hist_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                           if isinstance(self.attack[b][0], L.HistoryKind)]
        # the pairs whose attacker runs an ARC-aware attack (kind L.ArcAttackKind): the history or pipeline search
        # through the receiver's whole chain, its clipping step included (rcmarl_history_arc_attack /
        # rcmarl_pipeline_arc_attack); launches of their own, after the history ones (_arc_job_groups)
        self.arc_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                          if isinstance(self.attack[b][0], L.ArcAttackKind)]
        # the pairs whose attacker runs a subset-aware attack (kind L.SubsetAttackKind): against an mda / smea receiver
        # the history or pipeline search through its whole chain and its subset selection
        # (rcmarl_subset_history_attack / rcmarl_subset_pipeline_attack), against any other exactly an ARC pair's job;
        # launches of their own, after the ARC ones (_subset_job_groups)
        self.subset_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                             if isinstance(self.attack[b][0], L.SubsetAttackKind)]
        # the pairs whose attacker runs an IOS-aware attack (kind L.IosAttackKind): against an ios receiver the history
        # or pipeline search through its whole chain and its iterative outlier scissor (rcmarl_ios_history_attack /
        # rcmarl_ios_pipeline_attack), against any other exactly a subset pair's job; launches of their own, after the
        # subset ones (_ios_job_groups)
        self.ios_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                          if isinstance(self.attack[b][0], L.IosAttackKind)]
        self.gamma_pairs = (self.adapt_pairs + self.tailor_pairs + self.pipe_pairs + self.hist_pairs + self.arc_pairs
                            + self.subset_pairs + self.ios_pairs)
        # the pairs whose attacker runs the dissensus attack (rcmarl_dissensus_attack) and those that run the mimic attack
        # (rcmarl_mimic_attack, whose direction state carries over between epochs and rounds): a launch each, after the
        # tailored one
        self.diss_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs)
                           if isinstance(self.attack[b][0], L.DissensusKind)]
        self.mimic_pairs = [e for e, (b, _, _) in enumerate(self.byz_pairs) if isinstance(self.attack[b][0], L.MimicKind)]

    def _receiver_nodes(self, j):
        """in_nodes[j] with each Byzantine neighbour replaced by the message row crafted for receiver j."""
        row = {b: self.NA + e for e, (b, r, _) in enumerate(self.byz_pairs) if r == j}
        return [row.get(k, k) for k in self.in_nodes[j]]

    def _momentum_nodes(self, j):
        """The message rows cooperative agent j's clipping step reads: its momentum rows if it has momentum, else
        _receiver_nodes(j)."""
        if self.momentum[j] is not None:
            return list(range(self.mom_row[j], self.mom_row[j] + len(self.in_nodes[j])))
        return self._receiver_nodes(j)

    def _clipped_nodes(self, j):
        """The message rows cooperative agent j's mixing step reads: its clipped rows if it clips, else
        _momentum_nodes(j)."""
        if self.clipping[j] is not None:
            return list(range(self.arc_row[j], self.arc_row[j] + len(self.in_nodes[j])))
        return self._momentum_nodes(j)

    def _rule_nodes(self, j):
        """The message rows cooperative agent j's rule reads: its mixed rows if it mixes, else its clipped rows if it
        clips, else its momentum rows if it has momentum, else _receiver_nodes(j)."""
        if self.mixing[j] is None:
            return self._clipped_nodes(j)
        return list(range(self.mix_row[j], self.mix_row[j] + L.mixed_rows(self.mixing[j], len(self.in_nodes[j]))))

    def neighbour_weights(self):
        """{cooperative agent i with a distance-based, the dnc, an mda / smea or the ios rule: float32 [2, n_in]}: the
        weight w_k its rule gave each in-neighbour (in_nodes[i] order, a Byzantine neighbour's entry standing for the
        message crafted for i) in the last epoch of the last update round; row 0 for the critic, row 1 for the
        team-reward net.  For an agent that mixes, the rule weighs the mixed messages (the n_out rows of a bucketing agent), and the entry
        is the effective weight w M of each in-neighbour.  For an agent with momentum, entry k is the weight of slot k's
        momentum row.  For an agent that clips, with w' that weight and c its clipping factors (clipping_factors), entry
        k >= 1 is w'_k c_k and entry 0 is w'_0 + sum_{k >= 1} w'_k (1 - c_k): a clipped row is x_0 + c_k (x_k - x_0)."""
        out = {}
        for agents, weights in ((self.vec_agents, self.vec_weights), (self.dnc_agents, self.dnc_weights),
                                (self.subset_agents, self.subset_weights), (self.ios_agents, self.ios_weights)):
            if not agents:
                continue
            w = weights.cpu().numpy()
            self.d2h_bytes += w.nbytes
            out.update({i: w[2 * q:2 * q + 2, :len(self._rule_nodes(i))].copy() for q, i in enumerate(agents)})
        if any(self.mixing[i] is not None for i in out):
            mix = self.mixing_matrices()
            for i in out:
                if i in mix:
                    out[i] = np.einsum("tk,tkl->tl", out[i].astype(np.float64), mix[i]).astype(np.float32)
        if any(self.clipping[i] is not None for i in out):
            clip = self.clipping_factors()
            for i in out:
                if i in clip:
                    w, c = out[i].astype(np.float64), clip[i].astype(np.float64)
                    eff = w * c
                    eff[:, 0] = w[:, 0] + (w[:, 1:] * (1.0 - c[:, 1:])).sum(1)
                    out[i] = eff.astype(np.float32)
        return out

    def clipping_factors(self):
        """{cooperative agent i that clips: float32 [2, n_in]}: the factors c_k of its clipping step (rcmarl_arc_clip;
        c_0 = 1, in_nodes[i] order) in the last epoch of the last update round; row 0 for the critic, row 1 for the
        team-reward net."""
        if not self.arc_agents:
            return {}
        c = self.arc_weights.cpu().numpy()
        self.d2h_bytes += c.nbytes
        return {i: c[2 * q:2 * q + 2, :len(self.in_nodes[i])].copy() for q, i in enumerate(self.arc_agents)}

    def mixing_matrices(self):
        """{cooperative agent i that mixes: float32 [2, n_out, n_in]}: the mixing matrix M of the last epoch of the last
        update round; [0] for the critic, [1] for the team-reward net.  For nnm n_out = n_in and M[k, l] = 1/|N_k| if
        in-neighbour l (in_nodes[i] order) is among the nearest of k and 0 otherwise (rcmarl_nnm_mix); for bucketing
        n_out = 1 + ceil((n_in - 1) / s), M[0, 0] = 1 and M[1 + b, l] = 1/|bucket b| if l is in bucket b
        (rcmarl_bucket_mix)."""
        if not self.mix_agents:
            return {}
        m = self.mix_weights.cpu().numpy()
        self.d2h_bytes += m.nbytes
        out = {}
        for q, i in enumerate(self.mix_agents):
            n, n_out = len(self.in_nodes[i]), len(self._rule_nodes(i))
            out[i] = m[2 * q:2 * q + 2, :n_out * n].reshape(2, n_out, n).copy()
        return out

    def attack_gammas(self):
        """{(attacker b, cooperative receiver j) of a min-max / min-sum, a tailored, a pipeline, a history, an ARC, a
        subset or an IOS attack: float32 [2]}: the gamma of the message b crafted for j in the last epoch of the last
        update round (include/rcmarl.h, rcmarl_adaptive_attack; for a tailored, pipeline, history, ARC, subset or IOS
        attack gamma_i*, rcmarl_tailored_attack / rcmarl_pipeline_attack / rcmarl_history_attack / their ARC, subset and
        IOS forms); entry 0 for the critic, 1 for the team-reward net."""
        if not self.gamma_pairs:
            return {}
        g = self.att_gamma.cpu().numpy()
        self.d2h_bytes += g.nbytes
        return {self.byz_pairs[e][:2]: g[q].copy() for q, e in enumerate(self.gamma_pairs)}

    def mimic_targets(self):
        """{(attacker b, cooperative receiver j) of a mimic attack: int32 [2]}: the agent whose message b copied for j in
        the last epoch of the last update round (include/rcmarl.h, rcmarl_mimic_attack); entry 0 for the critic, 1 for
        the team-reward net."""
        if not self.mimic_pairs:
            return {}
        k = self.mimic_target.cpu().numpy()
        self.d2h_bytes += k.nbytes
        out = {}
        for q, e in enumerate(self.mimic_pairs):
            b, j, honest = self.byz_pairs[e]
            out[(b, j)] = np.array([honest[k[q, t]] for t in range(2)], np.int32)
        return out

    def _tailored_slots(self, j):
        """(slots, honest) of receiver j for rcmarl_tailored_attack: _receiver_nodes(j) with every Byzantine pair row
        replaced by -1 (a crafted slot), and the indices of the cooperative slots."""
        slots = [-1 if r >= self.NA else r for r in self._receiver_nodes(j)]
        honest = [k for k, i in enumerate(self.in_nodes[j]) if self.labels[i] == COOP]
        return slots, honest

    def _arc_staging(self, j, n_real, kc):
        """(floats, bound) of the job an ARC pair against receiver j gets (include/rcmarl.h): the history form's
        (n_in + 4 + (DnC or IOS ? 2 : 0) + k_clip) * PT if j has momentum, else the pipeline form's (n_real + n_mixed +
        4 + (DnC or IOS ? 2 : 0) + k_clip) * PT, with k_clip = kc (0 when j does not clip)."""
        n_in, extra = len(self.in_nodes[j]), (2 if self.dnc[j] or self.ios[j] else 0) + 4 + kc
        PT = L.param_count(3 * self.NA, 1)             # the TR net, the larger of the two
        if self.momentum[j] is not None:
            return (n_in + extra) * PT, L.HISTORY_MAX_FLOATS
        mix = self.mixing[j]
        n_mixed = 0 if mix is None else n_in if mix == "nnm" else L.mixed_rows(mix, n_in) - 1
        return (n_real + n_mixed + extra) * PT, L.PIPELINE_MAX_FLOATS

    def _arc_job_groups(self):
        """The job tables of the ARC pairs' messages update_round launches in every epoch, after the history
        launches: a list of (launch, group, mom), each group of at most MAX_JOBS jobs, with mom the momentum agent index
        of each job of a history-form group (its `first` is set per epoch) and None for a pipeline-form group (its
        `epoch` is set per epoch).  Per pair one critic and one TR job: against a receiver that clips, the history form
        (momentum) or the pipeline form (with the receiver's mixing) through its clipping step; against one that does
        not, exactly the job a history pair gets."""
        n_before = len(self.adapt_pairs) + len(self.tailor_pairs) + len(self.pipe_pairs) + len(self.hist_pairs)
        return self._chain_job_groups(self.arc_pairs, n_before)

    def _subset_job_groups(self):
        """_arc_job_groups for the subset pairs, launched after the ARC groups: against an mda / smea receiver the
        history form (momentum) or the pipeline form (with the receiver's mixing) of rcmarl_subset_history_attack /
        rcmarl_subset_pipeline_attack, with arc = whether the receiver clips (the launch is functools.partial of
        ops.subset_history_attack / ops.subset_pipeline_attack with that arc); against any other receiver exactly the
        job, and the launch, an ARC pair gets."""
        n_before = (len(self.adapt_pairs) + len(self.tailor_pairs) + len(self.pipe_pairs) + len(self.hist_pairs)
                    + len(self.arc_pairs))
        return self._chain_job_groups(self.subset_pairs, n_before)

    def _ios_job_groups(self):
        """_arc_job_groups for the IOS pairs, launched after the subset groups: against an ios receiver the history form
        (momentum) or the pipeline form (with the receiver's mixing) of rcmarl_ios_history_attack /
        rcmarl_ios_pipeline_attack, with arc = whether the receiver clips (the launch is functools.partial of
        ops.ios_history_attack / ops.ios_pipeline_attack with that arc); against an mda / smea receiver exactly the job,
        and the launch, a subset pair gets; against any other exactly those an ARC pair gets."""
        n_before = (len(self.adapt_pairs) + len(self.tailor_pairs) + len(self.pipe_pairs) + len(self.hist_pairs)
                    + len(self.arc_pairs) + len(self.subset_pairs))
        return self._chain_job_groups(self.ios_pairs, n_before)

    def _chain_job_groups(self, pairs, n_before):
        """The groups of _arc_job_groups / _subset_job_groups / _ios_job_groups for `pairs`, whose gamma rows start at
        n_before."""
        NA = self.NA
        mom_index = {i: q for q, i in enumerate(self.mom_agents)}
        tables = {}                                    # (ios rule, subset rule, history form, clips) -> ([jobs], [mom])
        for q_pair, e in enumerate(pairs):
            b, j, _ = self.byz_pairs[e]
            kind, param = self.attack[b]
            slots, hon = self._tailored_slots(j)
            subset, ios = self.subset_rule[j] is not None, self.ios[j]
            rule = ((L.TAILOR_SUBSET, self.subset_rule[j]) if subset
                    else (L.TAILOR_FILTER, L.FILTER_IOS) if ios
                    else (L.TAILOR_VECTOR, self.vector_rule[j]) if self.vector_rule[j] is not None
                    else (L.TAILOR_SPECTRAL, L.SPECTRAL_DNC) if self.dnc[j]
                    else (L.TAILOR_COORD, self.aggregation[j]))
            hist = self.momentum[j] is not None
            jobs, moms = tables.setdefault((ios, subset, hist, self.clipping[j] is not None), ([], []))
            for t, (msgs, P, ref) in enumerate(((self.msg_c, self.PC, self.critic[j]), (self.msg_t, self.PT, self.tr[j]))):
                gamma_out = self.att_gamma[n_before + q_pair, t:t + 1]
                if hist:
                    q = mom_index[j]
                    own = [k for k, i in enumerate(self.in_nodes[j]) if i == b]
                    jobs.append(ops.history_attack_job(
                        msgs[NA + e], msgs, P, P, slots, hon, rule, self.H[j], kind, param, ref,
                        self.momentum_M[q, t], self.PT, self.momentum[j], 0, own, gamma_out=gamma_out))
                    moms.append(q)
                else:
                    jobs.append(ops.pipeline_attack_job(
                        msgs[NA + e], msgs, P, P, slots, hon, rule, self.H[j], kind, param, mixing=self.mixing[j],
                        n_perms=L.PIPELINE_PERMS, seed=self.seed, attacker=b, receiver=j, net=t,
                        round=self.episodes_done & 0xFFFFFFFF, gamma_out=gamma_out))
        launch = {(True, True): ops.history_arc_attack, (True, False): ops.history_attack,
                  (False, True): ops.pipeline_arc_attack, (False, False): ops.pipeline_attack}
        cls = {True: L.HistoryAttackJob, False: L.PipelineAttackJob}
        out = []
        for (ios, subset, hist, clips), (jobs, moms) in sorted(tables.items(), reverse=True):
            fn = (functools.partial(ops.ios_history_attack if hist else ops.ios_pipeline_attack, arc=clips) if ios
                  else functools.partial(ops.subset_history_attack if hist else ops.subset_pipeline_attack, arc=clips)
                  if subset else launch[(hist, clips)])
            for g in range(0, len(jobs), L.MAX_JOBS):
                out.append((fn, ops.job_array(cls[hist], jobs[g:g + L.MAX_JOBS]), moms[g:g + L.MAX_JOBS] if hist else None))
        return out

    def _attack_job_groups(self):
        """The job tables of the Byzantine messages update_round launches in every epoch, each in groups of MAX_JOBS:
        (attack, adaptive, tailored, pipeline, history, dissensus, mimic groups), with the history groups and the mimic
        groups as (index of their first job, group) pairs, hist_mom the momentum agent index of each history job, and
        mimic_t0 each mimic pair's T0."""
        NA, lab = self.NA, self.labels
        # Byzantine messages: per (attacker, receiver) pair one critic and one TR job, crafted anew in every epoch
        # (the min-max / min-sum pairs in a job list of their own, with the gamma of each message)
        # (and the tailored pairs in a third, against their receiver's own rule and H)
        # (and the pipeline pairs in a fourth, against their receiver's mixing step, rule and H)
        # (and the history pairs in a fifth, through their receiver's momentum; a history pair whose receiver has no
        # momentum joins the pipeline pairs with the same direction and scale)
        # (then the dissensus pairs, and the mimic pairs with their direction states)
        att_jobs, ada_jobs, tail_jobs, pipe_jobs, hist_jobs, diss_jobs, mimic_jobs = [], [], [], [], [], [], []
        ada_row = {e: q for q, e in enumerate(self.adapt_pairs)}
        tail_row = {e: len(self.adapt_pairs) + q for q, e in enumerate(self.tailor_pairs)}
        pipe_row = {e: len(self.adapt_pairs) + len(self.tailor_pairs) + q for q, e in enumerate(self.pipe_pairs)}
        n_before = len(self.adapt_pairs) + len(self.tailor_pairs) + len(self.pipe_pairs)
        hist_row = {e: n_before + q for q, e in enumerate(self.hist_pairs)}
        pipe_row.update({e: r for e, r in hist_row.items() if self.momentum[self.byz_pairs[e][1]] is None})
        hist_row = {e: r for e, r in hist_row.items() if e not in pipe_row}
        hist_mom = []                                  # the momentum agent index q of each history job
        mom_index = {i: q for q, i in enumerate(self.mom_agents)}
        diss_set = set(self.diss_pairs)
        mimic_row = {e: q for q, e in enumerate(self.mimic_pairs)}
        # their jobs are _arc_job_groups' / _subset_job_groups' / _ios_job_groups'
        arc_set = set(self.arc_pairs + self.subset_pairs + self.ios_pairs)
        for e, (b, j, honest) in enumerate(self.byz_pairs):
            if e in arc_set:
                continue
            kind, param = self.attack[b]
            if e in diss_set:
                # colluding dissensus attackers of j split the cancellation: n_byz counts their entries of in_nodes[j]
                n_byz = sum(isinstance(self.attack[k][0], L.DissensusKind) for k in self.in_nodes[j]
                            if lab[k] == BYZANTINE)
                for msgs, P in ((self.msg_c, self.PC), (self.msg_t, self.PT)):
                    diss_jobs.append(ops.dissensus_attack_job(msgs[NA + e], msgs, P, P, j, honest, n_byz, param))
                continue
            if e in mimic_row:
                # copying the receiver to itself only slows its consensus: the candidates are S_j without j's own
                # entries, unless that leaves none
                q = mimic_row[e]
                cand = [k for k, i in enumerate(honest) if i != j] or list(range(len(honest)))
                for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                    mimic_jobs.append(ops.mimic_attack_job(msgs[NA + e], msgs, P, P, honest, cand, self.mimic_z[q, t],
                                                           0, target_out=self.mimic_target[q, t:t + 1]))
                continue
            if e in tail_row or e in pipe_row or e in hist_row:
                slots, hon = self._tailored_slots(j)
                rule = ((L.TAILOR_VECTOR, self.vector_rule[j]) if self.vector_rule[j] is not None
                        else (L.TAILOR_SPECTRAL, L.SPECTRAL_DNC) if self.dnc[j]
                        else (L.TAILOR_COORD, self.aggregation[j]))
            if e in hist_row:
                q = mom_index[j]
                own = [k for k, i in enumerate(self.in_nodes[j]) if i == b]
                for t, (msgs, P, ref) in enumerate(((self.msg_c, self.PC, self.critic[j]),
                                                    (self.msg_t, self.PT, self.tr[j]))):
                    hist_jobs.append(ops.history_attack_job(
                        msgs[NA + e], msgs, P, P, slots, hon, rule, self.H[j], kind, param, ref,
                        self.momentum_M[q, t], self.PT, self.momentum[j], 0, own,
                        gamma_out=self.att_gamma[hist_row[e], t:t + 1]))
                    hist_mom.append(q)
                continue
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                if e in pipe_row:
                    pipe_jobs.append(ops.pipeline_attack_job(
                        msgs[NA + e], msgs, P, P, slots, hon, rule, self.H[j], kind, param, mixing=self.mixing[j],
                        n_perms=L.PIPELINE_PERMS, seed=self.seed, attacker=b, receiver=j, net=t,
                        round=self.episodes_done & 0xFFFFFFFF, gamma_out=self.att_gamma[pipe_row[e], t:t + 1]))
                elif e in tail_row:
                    tail_jobs.append(ops.tailored_attack_job(msgs[NA + e], msgs, P, P, slots, hon, rule, self.H[j], kind,
                                                             param, gamma_out=self.att_gamma[tail_row[e], t:t + 1]))
                elif e in ada_row:
                    ada_jobs.append(ops.adaptive_attack_job(msgs[NA + e], msgs, P, P, honest, kind, param,
                                                            gamma_out=self.att_gamma[ada_row[e], t:t + 1]))
                else:
                    att_jobs.append(ops.attack_job(msgs[NA + e], msgs, P, P, honest, kind, param, seed=self.seed,
                                                   attacker=b, receiver=j, round=self.episodes_done & 0xFFFFFFFF))
        att_groups = [ops.job_array(L.AttackJob, att_jobs[g:g + L.MAX_JOBS]) for g in range(0, len(att_jobs), L.MAX_JOBS)]
        ada_groups = [ops.job_array(L.AdaptiveAttackJob, ada_jobs[g:g + L.MAX_JOBS])
                      for g in range(0, len(ada_jobs), L.MAX_JOBS)]
        tail_groups = [ops.job_array(L.TailoredAttackJob, tail_jobs[g:g + L.MAX_JOBS])
                       for g in range(0, len(tail_jobs), L.MAX_JOBS)]
        pipe_groups = [ops.job_array(L.PipelineAttackJob, pipe_jobs[g:g + L.MAX_JOBS])
                       for g in range(0, len(pipe_jobs), L.MAX_JOBS)]
        hist_groups = [(g, ops.job_array(L.HistoryAttackJob, hist_jobs[g:g + L.MAX_JOBS]))
                       for g in range(0, len(hist_jobs), L.MAX_JOBS)]
        diss_groups = [ops.job_array(L.DissensusJob, diss_jobs[g:g + L.MAX_JOBS])
                       for g in range(0, len(diss_jobs), L.MAX_JOBS)]
        # mimic job 2q + t belongs to pair mimic_pairs[q]; its T0 is the attacker's parameter
        mimic_t0 = [int(self.attack[self.byz_pairs[e][0]][1]) for e in self.mimic_pairs]
        mimic_groups = [(g, ops.job_array(L.MimicJob, mimic_jobs[g:g + L.MAX_JOBS]))
                        for g in range(0, len(mimic_jobs), L.MAX_JOBS)]
        return (att_groups, ada_groups, tail_groups, pipe_groups, hist_groups, hist_mom, diss_groups, mimic_t0,
                mimic_groups)

    def _try_peer_comm(self):
        """Set up the peer-memory exchange on every rank, or on none: the ranks agree (MIN all-reduce of a success
        flag) so that a box without IPC / peer access falls back to the NCCL path consistently instead of deadlocking."""
        import torch.distributed as dist
        from .comm import PeerComm
        comm, ok = None, 1
        try:
            comm = PeerComm(self.rank, self.world, self.group)
        except Exception as ex:                                      # noqa: BLE001 -- any failure means "use NCCL"
            ok = 0
            if self.rank == 0:
                print(f"[rcmarl] peer-memory exchange unavailable ({ex}); using NCCL all-reduce", flush=True)
        flag = torch.tensor([ok], device=self.dev, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            if comm is not None:
                comm.close()
            return None
        return comm

    def _allreduce(self, t):
        """Sum the packed gradient sums over ranks -- unless the bound peer-memory context already did it in-kernel."""
        if self.comm is not None:
            return t
        return dist_util.allreduce_sums(t, self.world, self.group)

    def _timed(self, name, fn, *args):
        """Run fn(*args); when profiling is on, bracket it with CUDA events on the launching stream."""
        if self.profile is None:
            return fn(*args)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(*args)
        b.record()
        self.profile.setdefault(name, []).append((a, b))

    def _perm(self, T):
        if self.perm_source is not None:
            p = np.asarray(self.perm_source(T), np.int32)
            assert p.shape == (T,)
            return torch.as_tensor(p)
        return torch.randperm(T, generator=self._perm_gen, dtype=torch.int32)

    def _rows(self, row_begin, n_rows, time_idx=None):
        return ops.make_rows(self.sa, self.ns, self.r, self.NA, row_begin, n_rows, time_idx, self.N)

    def get_weights(self, i):
        """[actor, critic, TR(, critic_local)] as Keras weight lists (get_parameters, res..py:221-223)."""
        NA, n = self.NA, self.n_real
        self.d2h_bytes += 4 * (self.PA + self.PC + self.PT + (self.PC if self.labels[i] == MALICIOUS else 0))
        out = [nets.unpack_padded(self.actor[i].cpu().numpy(), 2 * n, 2 * NA, 5),
               nets.unpack_padded(self.critic[i].cpu().numpy(), 2 * n, 2 * NA, 1),
               nets.unpack_padded(self.tr[i].cpu().numpy(), 3 * n, 3 * NA, 1)]
        if self.labels[i] == MALICIOUS:
            out.append(nets.unpack_padded(self.critic_local[i].cpu().numpy(), 2 * n, 2 * NA, 1))
        return out

    # ------------------------------------------------------------------ rollout
    def rollout_block(self, n_episodes=None, uniforms=None, init_state=None):
        """Episodes under the current (fixed) policy for all environments: ONE kernel launch
        (train_agents.py:46-80).  Returns per-episode means over this rank's environments:
        est[n_ep, NA] (critic(state_0), :60-62) and ret[n_ep, NA] (discounted returns, :71)."""
        n_ep = self.n_ep_fixed if n_episodes is None else int(n_episodes)
        Lq = self.max_ep_len
        if self.t_filled + n_ep * Lq > self.Tcap:
            raise L.RcmarlError("replay buffer overflow: call update_round() (which trims) before the next block")
        est = torch.empty(n_ep, self.N, self.NA, dtype=torch.float32, device=self.dev)
        ret = torch.empty(n_ep, self.N, self.NA, dtype=torch.float32, device=self.dev)
        self._timed("rollout", self._rollout_launch, est, ret, n_ep, uniforms, init_state)
        self.launches += 1
        self.t_filled += n_ep * Lq
        self.episodes_done += n_ep
        stats = torch.empty(2, n_ep, self.NA, dtype=torch.float32, device=self.dev)
        ops.episode_means(est, stats[0])                                   # logging only (train_agents.py:168-180)
        ops.episode_means(ret, stats[1])
        self.launches += 2
        if self.world > 1:
            dist_util.allreduce_sums(stats, self.world, self.group)     # logging only (NCCL)
            stats /= self.world
        stats = stats.cpu().numpy()[:, :, :self.n_real]
        self.d2h_bytes += stats.nbytes
        return stats[0], stats[1]

    def _rollout_launch(self, est, ret, n_ep, uniforms, init_state):
        Lq = self.max_ep_len
        if init_state is None and self.fixed_initial_state is not None:    # randomize_state=False: every reset -> initial_state
            if self._fixed_init_dev is None or self._fixed_init_dev.shape[0] < n_ep:
                host = np.broadcast_to(self.fixed_initial_state, (n_ep, self.N, self.NA, 2))
                self._fixed_init_dev = torch.as_tensor(np.ascontiguousarray(host)).to(self.dev)
            init_state = self._fixed_init_dev
        ops.rollout(self.actor, self.critic, self.desired, self.sa, self.ns, self.r, self.t_filled, est, ret,
                    n_envs=self.N, n_agents=self.NA, n_episodes=n_ep, max_ep_len=Lq, nrow=self.nrow, ncol=self.ncol,
                    n_active=self.n_real, gamma=self.gamma, mu=self.mu, seed=self.seed, env_offset=self.rank * self.N,
                    episode_offset=self.episodes_done, uniforms=uniforms, init_state=init_state, scaling=self.scaling)

    def load_rows(self, s, ns, a, r):
        """Append externally produced transitions (exp_buffer, train_agents.py:36-40; parity tests; bench e2e).
        s, ns: (B, NA, 2); a, r: (B, NA, 1) as lists / NumPy arrays / (pinned) host or device torch tensors;
        B must be a multiple of n_envs, rows time-major.  The sa = concat([s, a]) of train_agents.py:93 is formed by
        strided device copies (data movement only)."""
        n = self.n_real

        def t(x, last):
            if not isinstance(x, torch.Tensor):
                x = torch.as_tensor(np.asarray(x, np.float32))
            return x.reshape(-1, n, last)
        s, ns, a, r = t(s, 2), t(ns, 2), t(a, 1), t(r, 1)
        B = s.shape[0]
        assert B % self.N == 0 and self.t_filled * self.N + B <= self.Tcap * self.N
        o = self.t_filled * self.N
        sa3 = self.sa.view(-1, self.NA, 3)                      # unused agent slots stay zero (the buffers start zeroed)
        sa3[o:o + B, :n, :2].copy_(s.to(self.dev, dtype=torch.float32, non_blocking=True))
        sa3[o:o + B, :n, 2:].copy_(a.to(self.dev, dtype=torch.float32, non_blocking=True))
        self.ns.view(-1, self.NA, 2)[o:o + B, :n].copy_(ns.to(self.dev, dtype=torch.float32, non_blocking=True))
        self.r.view(-1, self.NA, 1)[o:o + B, :n].copy_(r.to(self.dev, dtype=torch.float32, non_blocking=True))
        self.h2d_bytes += 4 * B * n * 6
        self.t_filled += B // self.N

    # ------------------------------------------------------------------ update round
    def update_round(self):
        """training/train_agents.py:86-163 for all agents and all local environments."""
        NA, N, T = self.NA, self.N, self.t_filled
        B = T * N
        Bg = B * self.world
        lab = self.labels
        coop = self.coop
        mal = [i for i in range(NA) if lab[i] == MALICIOUS]
        rows_all = self._rows(0, B)
        r_col = [self.r[:, i] for i in range(NA)]

        if coop:                                                           # :96-98
            ops.reward_mix(self.r[:B], coop, out=self.r_coop, scale=1.0)
            self.launches += 1
            if mal:
                ops.reward_mix(self.r[:B], coop, out=self.neg_r_coop, scale=-1.0)
                self.launches += 1

        def applied(i):                                                    # r_applied, :106
            return (self.r_coop, 1) if self.common_reward else (r_col[i], NA)

        # ---- job tables that do not change across epochs
        td_jobs = []
        for i in range(NA):
            if lab[i] == COOP:
                add, st = applied(i)
                td_jobs.append(ops.value_job(self.tdt[i], [(self.critic[i], L.IN_NS, self.gamma)], add=add, add_stride=st))
            elif lab[i] == GREEDY:
                td_jobs.append(ops.value_job(self.tdt[i], [(self.critic[i], L.IN_NS, self.gamma)], add=r_col[i], add_stride=NA))
            elif lab[i] == MALICIOUS:
                k = mal.index(i)
                td_jobs.append(ops.value_job(self.tdt_local[k], [(self.critic_local[i], L.IN_NS, self.gamma)],
                                             add=r_col[i], add_stride=NA))                       # adversarial:148-149
                td_jobs.append(ops.value_job(self.tdt[i], [(self.critic[i], L.IN_NS, self.gamma)],
                                             add=self.neg_r_coop, add_stride=1))                 # adversarial:131-132
        td_arr = ops.job_array(L.ValueJob, td_jobs)

        fit_first, fit_next, fit_apply_first, fit_apply_next = [], [], [], []
        for n, i in enumerate(coop):
            lr2 = self.fast_lr[i] * 2.0 / Bg
            tgt_t, st_t = applied(i)
            sc, stt = self.sums_fit[2 * n][:self.PC + 1], self.sums_fit[2 * n + 1]
            for first in (True, False):
                wc = self.critic[i] if first else self.msg_c[i]
                wt = self.tr[i] if first else self.msg_t[i]
                gj = [ops.grad_job(wt, tgt_t, stt, L.IN_SA, target_stride=st_t),
                      ops.grad_job(wc, self.tdt[i], sc, L.IN_S)]
                aj = [ops.sgd_job(self.msg_t[i], wt, stt, self.PT, lr2, loss_out=self.loss_t[i:i + 1] if first else None,
                                  loss_coef=1.0 / Bg),
                      ops.sgd_job(self.msg_c[i], wc, sc, self.PC, lr2, loss_out=self.loss_c[i:i + 1] if first else None,
                                  loss_coef=1.0 / Bg)]
                (fit_first if first else fit_next).extend(gj)
                (fit_apply_first if first else fit_apply_next).extend(aj)
        fit_first, fit_next = ops.job_array(L.GradJob, fit_first), ops.job_array(L.GradJob, fit_next)
        fit_apply_first, fit_apply_next = ops.job_array(L.SgdJob, fit_apply_first), ops.job_array(L.SgdJob, fit_apply_next)

        # mini-batch chains of the adversaries (adversarial:133,150,163,239,251), node order = permutation order
        chains = []                                       # (weights in place, kind, target, stride, loss slot, lr)
        for i in range(NA):
            lr_i = self.fast_lr[i]
            if lab[i] == MALICIOUS:
                k = mal.index(i)
                chains.append((self.critic_local[i], L.IN_S, self.tdt_local[k], 1, None, lr_i))
                chains.append((self.tr[i], L.IN_SA, self.neg_r_coop, 1, self.loss_t[i:i + 1], lr_i))
                chains.append((self.critic[i], L.IN_S, self.tdt[i], 1, self.loss_c[i:i + 1], lr_i))
            elif lab[i] == GREEDY:
                chains.append((self.tr[i], L.IN_SA, r_col[i], NA, self.loss_t[i:i + 1], lr_i))
                chains.append((self.critic[i], L.IN_S, self.tdt[i], 1, self.loss_c[i:i + 1], lr_i))

        cons_jobs, team_jobs, team_apply = [], [], []
        for n, i in enumerate(coop):
            agg_row = self.vec_row.get(i, self.dnc_row.get(i, self.subset_row.get(i, self.ios_row.get(i))))
            if agg_row is not None:                        # the aggregate as the single in-node: clip returns it exactly
                nodes, H, rule = [agg_row], 0, L.AGG_CLIP
            else:
                nodes, H, rule = self._rule_nodes(i), self.H[i], self.aggregation[i]
            cons_jobs.append(ops.consensus_job(self.critic[i], self.msg_c, self.PC, nets.n_hidden_params(2 * NA), nodes, H, rule))
            cons_jobs.append(ops.consensus_job(self.tr[i], self.msg_t, self.PT, nets.n_hidden_params(3 * NA), nodes, H, rule))
            team_jobs.append(ops.team_job(self.critic[i], L.IN_S, self.msg_c, self.PC, nodes, H, sums=self.sums_team[2 * n], rule=rule))
            team_jobs.append(ops.team_job(self.tr[i], L.IN_SA, self.msg_t, self.PT, nodes, H, sums=self.sums_team[2 * n + 1], rule=rule))
            team_apply.append(ops.sgd_job(self.critic[i], self.critic[i], self.sums_team[2 * n], self.PC, -1.0 / Bg, first=self.PC - 21))
            team_apply.append(ops.sgd_job(self.tr[i], self.tr[i], self.sums_team[2 * n + 1], self.PT, -1.0 / Bg, first=self.PT - 21))
        cons_jobs, team_jobs = ops.job_array(L.ConsensusJob, cons_jobs), ops.job_array(L.TeamJob, team_jobs)
        team_apply = ops.job_array(L.SgdJob, team_apply)

        # the Byzantine messages' job tables (_attack_job_groups)
        (att_groups, ada_groups, tail_groups, pipe_groups, hist_groups, hist_mom, diss_groups, mimic_t0,
         mimic_groups) = self._attack_job_groups()
        arc_groups = self._arc_job_groups() + self._subset_job_groups() + self._ios_job_groups()

        # the mixed rows of the agents that mix, from the messages each hears (crafted Byzantine ones included): at most
        # 16 cooperative agents x 2 nets, so one nnm launch and one bucketing launch per epoch.  A bucketing job draws
        # its permutation from (seed, round, epoch, receiver, net), so every epoch buckets anew and every rank of a
        # data-parallel run draws the same buckets.
        mix_jobs, bucket_jobs = [], []
        for q, i in enumerate(self.mix_agents):
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                if L.is_bucket_mixing(self.mixing[i]):
                    bucket_jobs.append(ops.bucket_job(msgs[self.mix_row[i]], msgs, P, P, self._clipped_nodes(i),
                                                      self.mixing[i][1], seed=self.seed, receiver=i, net=t,
                                                      round=self.episodes_done & 0xFFFFFFFF,
                                                      weights_out=self.mix_weights[2 * q + t]))
                else:
                    mix_jobs.append(ops.vector_job(msgs[self.mix_row[i]], msgs, P, P, self._clipped_nodes(i),
                                                   self.H[i], L.MIX_NNM, weights_out=self.mix_weights[2 * q + t]))
        mix_jobs = ops.job_array(L.VectorJob, mix_jobs) if mix_jobs else None
        # the momentum rows of the agents with momentum against their nets after the last consensus step (critic[i] /
        # tr[i], which Phase I leaves untouched): at most 16 cooperative agents x 2 nets, so one launch per epoch
        mom_jobs = []
        for q, i in enumerate(self.mom_agents):
            for t, (msgs, P, ref) in enumerate(((self.msg_c, self.PC, self.critic[i]), (self.msg_t, self.PT, self.tr[i]))):
                mom_jobs.append(ops.momentum_job(msgs[self.mom_row[i]], msgs, P, P, self._receiver_nodes(i), ref,
                                                 self.momentum_M[q, t], self.PT, self.momentum[i], 0))
        mom_jobs = ops.job_array(L.MomentumJob, mom_jobs) if mom_jobs else None
        # the clipped rows of the agents that clip, from their momentum rows or the messages they hear: at most 16
        # cooperative agents x 2 nets, so one launch per epoch, after the momentum launch and before the mixing launches
        arc_jobs = []
        for q, i in enumerate(self.arc_agents):
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                arc_jobs.append(ops.vector_job(msgs[self.arc_row[i]], msgs, P, P, self._momentum_nodes(i), self.H[i],
                                               L.MIX_ARC, weights_out=self.arc_weights[2 * q + t]))
        arc_jobs = ops.job_array(L.VectorJob, arc_jobs) if arc_jobs else None

        def momentum_step():
            if mom_jobs is not None:                                       # job 2q + t belongs to mom_agents[q]
                for k, job in enumerate(mom_jobs):
                    job.first = int(self.momentum_steps[k // 2] == 0)
                ops.momentum_mix(mom_jobs)
                self.launches += 1
                self.momentum_steps = [s + 1 for s in self.momentum_steps]
        bucket_groups = [ops.job_array(L.BucketJob, bucket_jobs[g:g + L.MAX_JOBS])
                         for g in range(0, len(bucket_jobs), L.MAX_JOBS)]
        # distance-based aggregates over the messages each receiver hears (or their mixed rows): at most 16
        # cooperative agents x 2 nets, so one launch per epoch
        vec_jobs = []
        for q, i in enumerate(self.vec_agents):
            nodes, row = self._rule_nodes(i), self.vec_row[i]
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                vec_jobs.append(ops.vector_job(msgs[row], msgs, P, P, nodes, self.H[i], self.vector_rule[i],
                                               weights_out=self.vec_weights[2 * q + t]))
        vec_jobs = ops.job_array(L.VectorJob, vec_jobs) if vec_jobs else None
        # the dnc aggregates likewise, in one launch of their own
        dnc_jobs = []
        for q, i in enumerate(self.dnc_agents):
            nodes, row = self._rule_nodes(i), self.dnc_row[i]
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                dnc_jobs.append(ops.vector_job(msgs[row], msgs, P, P, nodes, self.H[i], L.SPECTRAL_DNC,
                                               weights_out=self.dnc_weights[2 * q + t]))
        dnc_jobs = ops.job_array(L.VectorJob, dnc_jobs) if dnc_jobs else None
        # the mda / smea aggregates likewise, in one launch of their own
        subset_jobs = []
        for q, i in enumerate(self.subset_agents):
            nodes, row = self._rule_nodes(i), self.subset_row[i]
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                subset_jobs.append(ops.vector_job(msgs[row], msgs, P, P, nodes, self.H[i], self.subset_rule[i],
                                                  weights_out=self.subset_weights[2 * q + t]))
        subset_jobs = ops.job_array(L.VectorJob, subset_jobs) if subset_jobs else None
        # the ios aggregates likewise, in one launch of their own
        ios_jobs = []
        for q, i in enumerate(self.ios_agents):
            nodes, row = self._rule_nodes(i), self.ios_row[i]
            for t, (msgs, P) in enumerate(((self.msg_c, self.PC), (self.msg_t, self.PT))):
                ios_jobs.append(ops.vector_job(msgs[row], msgs, P, P, nodes, self.H[i], L.FILTER_IOS,
                                               weights_out=self.ios_weights[2 * q + t]))
        ios_jobs = ops.job_array(L.VectorJob, ios_jobs) if ios_jobs else None

        for epoch in range(self.n_epochs):                                 # :100
            # ---------------- I) local updates (:105-121)
            if td_jobs:
                ops.values(rows_all, td_arr)
                self.launches += 1
            if coop:
                for step in range(self.local_steps):                      # fit(batch_size=B, epochs=5), res..py:118,136
                    self._timed("fit_grad", ops.grad, rows_all, fit_first if step == 0 else fit_next, L.LOSS_MSE, self.ws)
                    self._allreduce(self.sums_fit[:2 * len(coop)])
                    ops.sgd_apply(fit_apply_first if step == 0 else fit_apply_next)
                    self.launches += 3
            if chains:
                self._timed("minibatch_sgd", self._minibatch_sgd, chains, T)
            for i in range(self.n_real):                                   # the transmitted messages (:118-121)
                if lab[i] != COOP:
                    self.msg_c[i].copy_(self.critic[i])
                    self.msg_t[i].copy_(self.tr[i])
            for g in att_groups:
                for job in g:
                    job.epoch = epoch
                ops.attack(g)
                self.launches += 1
            for g in ada_groups:                                           # no epoch dependence: no job changes
                ops.adaptive_attack(g)
                self.launches += 1
            for g in tail_groups:                                          # no epoch dependence either
                ops.tailored_attack(g)
                self.launches += 1
            for g in pipe_groups:                                          # a bucketing receiver's samples per epoch
                for job in g:
                    job.epoch = epoch
                ops.pipeline_attack(g)
                self.launches += 1
            for g0, g in hist_groups:                                      # M as it stands before this epoch's step
                for k, job in enumerate(g):
                    job.first = int(self.momentum_steps[hist_mom[g0 + k]] == 0)
                ops.history_attack(g)
                self.launches += 1
            for launch, g, mom in arc_groups:                             # as the pipeline and history groups
                for k, job in enumerate(g):
                    if mom is None:
                        job.epoch = epoch
                    else:
                        job.first = int(self.momentum_steps[mom[k]] == 0)
                launch(g)
                self.launches += 1
            for g in diss_groups:                                          # no epoch dependence either
                ops.dissensus_attack(g)
                self.launches += 1
            if mimic_groups:                                               # a power step in each pair's first T0 epochs
                update = [int(s < t0) for s, t0 in zip(self.mimic_steps, mimic_t0)]
                for g0, g in mimic_groups:
                    for k, job in enumerate(g):
                        job.update = update[(g0 + k) // 2]
                    ops.mimic_attack(g)
                    self.launches += 1
                self.mimic_steps = [s + u for s, u in zip(self.mimic_steps, update)]
            # momentum, clipping and mixing touch disjoint agents' rows except momentum -> clipping -> mixing of an
            # agent that clips, so without one the momentum launch keeps its place after the mixing launches
            if arc_jobs is not None:
                momentum_step()
                ops.arc_clip(arc_jobs)
                self.launches += 1
            if mix_jobs is not None:
                ops.nnm_mix(mix_jobs)
                self.launches += 1
            for g in bucket_groups:
                for job in g:
                    job.epoch = epoch
                ops.bucket_mix(g)
                self.launches += 1
            if arc_jobs is None:
                momentum_step()
            if vec_jobs is not None:
                ops.vector_aggregate(vec_jobs)
                self.launches += 1
            if dnc_jobs is not None:
                ops.dnc_aggregate(dnc_jobs)
                self.launches += 1
            if subset_jobs is not None:
                ops.subset_aggregate(subset_jobs)
                self.launches += 1
            if ios_jobs is not None:
                ops.ios_aggregate(ios_jobs)
                self.launches += 1
            # ---------------- II) resilient consensus (:125-145)
            if coop:
                ops.consensus_hidden(cons_jobs)
                self._timed("team", ops.team, rows_all, team_jobs, self.ws)
                self._allreduce(self.sums_team[:2 * len(coop)])
                ops.sgd_apply(team_apply)
                # consensus_hidden + team_kernel per input kind (critic / team-reward nets) + reduce + sgd
                self.launches += 3 + len({j.kind for j in team_jobs})

        # ---------------- III) actor updates (:149-153) on the newest block
        Ta = min(self.block, T)
        a0 = (T - Ta) * N
        rows_act = self._rows(a0, Ta * N)
        d_jobs = []
        for i in range(self.n_real):
            if lab[i] == COOP:                                             # res..py:95-98
                d_jobs.append(ops.value_job(self.delta[i], [(self.tr[i], L.IN_SA, 1.0), (self.critic[i], L.IN_NS, self.gamma),
                                                            (self.critic[i], L.IN_S, -1.0)]))
            else:                                                          # adversarial:38-40,113-115,221-223
                cw = self.critic_local[i] if lab[i] == MALICIOUS else self.critic[i]
                d_jobs.append(ops.value_job(self.delta[i], [(cw, L.IN_NS, self.gamma), (cw, L.IN_S, -1.0)],
                                            add=r_col[i], add_stride=NA))
        ops.values(rows_act, ops.job_array(L.ValueJob, d_jobs))
        self.launches += 1
        Bag = Ta * N * self.world
        if coop:
            gj, aj = [], []
            for n, i in enumerate(coop):
                self.adam_t[i] += 1
                gj.append(ops.grad_job(self.actor[i], self.delta[i], self.sums_actor[n], L.IN_S, action_agent=i))
                aj.append(ops.adam_job(self.actor[i], self.adam_m[i], self.adam_v[i], self.sums_actor[n], self.PA, 1.0 / Bag,
                                       ops.keras_adam_lr_t(self.slow_lr[i], self.adam_t[i]), loss_out=self.loss_a[i:i + 1],
                                       loss_coef=1.0 / Bag))
            ops.grad(rows_act, ops.job_array(L.GradJob, gj), L.LOSS_CE, self.ws)
            self._allreduce(self.sums_actor[:len(coop)])
            ops.adam_apply(ops.job_array(L.AdamJob, aj))
            self.launches += 3
        adv = [i for i in range(self.n_real) if lab[i] != COOP]
        if adv:
            self._minibatch_adam(adv, T, Ta, a0)

        n = self.n_real
        losses = dict(critic_loss=self.loss_c.cpu().numpy().astype(np.float64)[:n],
                      TR_loss=self.loss_t.cpu().numpy().astype(np.float64)[:n],
                      actor_loss=self.loss_a.cpu().numpy().astype(np.float64)[:n])
        self.d2h_bytes += 3 * 8 * NA
        # ---------------- IV) buffer trim (:158-163)
        self.trim()
        return losses

    def _minibatch_sgd(self, chains, T):
        """10 epochs x ceil(T/32) sequential SGD steps per chain; a mini-batch = 32 time rows x all environments
        (Appendix C).  The chains advance in lock-step in ONE persistent kernel, or, data-parallel without the
        peer-memory exchange, as rcmarl_grad -> NCCL all-reduce -> rcmarl_sgd_apply per step.  Both take at most
        MAX_JOBS chains, and a team of 16 adversaries has up to 48: the chains, which are independent, then run in
        consecutive groups of MAX_JOBS."""
        E = self.mb_epochs
        # every permutation is drawn before the first group runs, chain-major (the order of the reference's fits)
        perms = torch.stack([torch.stack([self._perm(T) for _ in range(E)]) for _ in chains]).to(self.dev)  # [C,E,T]
        self.h2d_bytes += 4 * perms.numel()
        gj, aj = [], []
        for c, (w, kind, tgt, st, loss, lr) in enumerate(chains):
            n = self.PT if kind == L.IN_SA else self.PC
            sums = self.sums_mb[c][:n + 1]
            gj.append(ops.grad_job(w, tgt, sums, kind, target_stride=st, time_idx=perms[c]))
            aj.append(ops.sgd_job(w, w, sums, n, lr, loss_out=loss, loss_coef=1.0 / (T * self.N * self.world)))
        rows = self._rows(0, 0, perms)
        lrs = [ch[5] for ch in chains]
        for g0 in range(0, len(chains), L.MAX_JOBS):
            g = slice(g0, g0 + L.MAX_JOBS)
            if self.world == 1 or self.comm is not None:
                ops.minibatch_fit(rows, gj[g], aj[g], E, T, self.mb_times, lrs[0], self.mb_cells)
                self.launches += 1
            else:
                ops.minibatch_steps(rows, gj[g], aj[g], E, T, self.mb_times, lrs[g], self.world,
                                    lambda s=self.sums_mb[g]: self._allreduce(s), self.ws)
                self.launches += 3 * E * ((T + self.mb_times - 1) // self.mb_times)

    def _minibatch_adam(self, adv, T, Ta, a0):
        """actor.fit(batch_size=200, epochs=1) of the adversaries (adversarial:41,116,224)."""
        perms = torch.stack([self._perm(Ta) for _ in adv]).to(self.dev)    # [A, Ta], indices inside the actor window
        self.h2d_bytes += 4 * perms.numel()
        gj, aj = [], []
        for n, i in enumerate(adv):
            gj.append(ops.grad_job(self.actor[i], self.delta[i], self.sums_actor[n], L.IN_S, action_agent=i, time_idx=perms[n]))
            aj.append(ops.adam_job(self.actor[i], self.adam_m[i], self.adam_v[i], self.sums_actor[n], self.PA, 0.0, 0.0,
                                   loss_out=self.loss_a[i:i + 1], loss_coef=1.0 / (Ta * self.N * self.world), loss_accumulate=1))
            self.loss_a[i:i + 1].zero_()
        steps = ops.adam_minibatch_steps(self._rows(a0, 0, perms), gj, aj, Ta, self.actor_mb_times,
                                         [self.slow_lr[i] for i in adv], [self.adam_t[i] for i in adv], self.world,
                                         lambda: self._allreduce(self.sums_actor[:len(adv)]), self.ws)
        for i in adv:
            self.adam_t[i] += steps
        self.launches += 3 * steps

    # ------------------------------------------------------------------ checkpoint / resume
    def state_dict(self, include_buffer=True):
        """Everything needed to continue training bit-for-bit: parameters, Keras-Adam slots and step counts, the
        replay buffer, the episode counter that keys the Philox streams and the shuffle generator.  (The reference
        saves only the final weights, main.py:119-121; optimiser state and buffer are lost there -- SURVEY 5.)"""
        T = self.t_filled * self.N
        sd = dict(version=1, labels=list(self.labels), n_envs=self.N, t_filled=self.t_filled,
                  episodes_done=self.episodes_done, adam_t=list(self.adam_t), perm_rng=self._perm_gen.get_state(),
                  actor=self.actor.cpu(), critic=self.critic.cpu(), tr=self.tr.cpu(), critic_local=self.critic_local.cpu(),
                  adam_m=self.adam_m.cpu(), adam_v=self.adam_v.cpu())
        if include_buffer:
            sd.update(sa=self.sa[:T].cpu(), ns=self.ns[:T].cpu(), r=self.r[:T].cpu())
        if self.mimic_pairs:                       # the mimic attack's state carries over between rounds
            sd.update(mimic_z=self.mimic_z.cpu(), mimic_steps=list(self.mimic_steps))
        if getattr(self, "mom_agents", None):      # so does the momentum of the agents with momentum
            sd.update(momentum_M=self.momentum_M.cpu(), momentum_steps=list(self.momentum_steps))
        return sd

    def load_state_dict(self, sd):
        if list(sd["labels"]) != list(self.labels) or int(sd["n_envs"]) != self.N:
            raise L.RcmarlError("checkpoint was written for a different agent set / environment count")
        if self.mimic_pairs:
            if "mimic_z" not in sd or "mimic_steps" not in sd:
                raise L.RcmarlError("checkpoint holds no mimic attack state, and this trainer has mimic attackers")
            if tuple(sd["mimic_z"].shape) != tuple(self.mimic_z.shape) or len(sd["mimic_steps"]) != len(self.mimic_steps):
                raise L.RcmarlError(f"checkpointed mimic state of shape {tuple(sd['mimic_z'].shape)} does not match "
                                    f"this trainer's {tuple(self.mimic_z.shape)}")
        mom = getattr(self, "mom_agents", None)    # (state_dict and load_state_dict read only the attributes they need)
        if mom:
            if "momentum_M" not in sd or "momentum_steps" not in sd:
                raise L.RcmarlError("checkpoint holds no momentum state, and this trainer has agents with momentum")
            if (tuple(sd["momentum_M"].shape) != tuple(self.momentum_M.shape)
                    or len(sd["momentum_steps"]) != len(self.momentum_steps)):
                raise L.RcmarlError(f"checkpointed momentum state of shape {tuple(sd['momentum_M'].shape)} does not "
                                    f"match this trainer's {tuple(self.momentum_M.shape)}")
        for name in ("actor", "critic", "tr", "critic_local", "adam_m", "adam_v"):
            getattr(self, name).copy_(sd[name])
        self.adam_t = [int(t) for t in sd["adam_t"]]
        self.episodes_done = int(sd["episodes_done"])
        self._perm_gen.set_state(sd["perm_rng"])
        if self.mimic_pairs:
            self.mimic_z.copy_(sd["mimic_z"])
            self.mimic_steps = [int(s) for s in sd["mimic_steps"]]
        if mom:
            self.momentum_M.copy_(sd["momentum_M"])
            self.momentum_steps = [int(s) for s in sd["momentum_steps"]]
        self.t_filled = 0
        if "sa" in sd:
            T = int(sd["t_filled"]) * self.N
            if T > self.sa.shape[0]:
                raise L.RcmarlError("checkpointed replay buffer does not fit")
            self.sa[:T].copy_(sd["sa"]); self.ns[:T].copy_(sd["ns"]); self.r[:T].copy_(sd["r"])
            self.t_filled = int(sd["t_filled"])

    def save(self, path, include_buffer=True):
        torch.save(self.state_dict(include_buffer), path)

    def load(self, path):
        self.load_state_dict(torch.load(path, map_location="cpu", weights_only=True))

    def trim(self):
        """Keep the newest `buffer_size` time rows (train_agents.py:158-163): chunked, non-overlapping
        device-to-device copies (pure data movement)."""
        q = self.t_filled - self.buffer_size
        if q <= 0:
            return
        N = self.N
        keep = self.buffer_size
        for buf in (self.sa, self.ns, self.r):
            done = 0
            while done < keep:
                n = min(q, keep - done)
                buf[done * N:(done + n) * N].copy_(buf[(done + q) * N:(done + q + n) * N])
                done += n
        self.t_filled = keep
