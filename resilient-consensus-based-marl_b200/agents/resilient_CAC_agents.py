"""RPBCAC_agent with the reference's API (agents/resilient_CAC_agents.py:5-223 of
mfigura/Resilient-consensus-based-MARL), executed by the sm_90a kernels of librcmarl.so.

Same constructor and method names, argument meaning and mutation conventions as the reference (SURVEY.md 8b):
  *_update_local            return (message copy, loss) and leave the agent's own networks untouched (:113,120)
  resilient_consensus_*_hidden   overwrite the hidden layers with the clipped mean of the neighbours' (:142-166), or
                                 their trimmed / W-MSR mean with aggregation="trim" / "wmsr", or the hidden layers
                                 of a distance-based ("krum", "mkrum", "scclip", "gmed"), divide-and-conquer
                                 ("dnc"), exact subset-selection ("mda", "smea") or iterative outlier scissor ("ios")
                                 aggregate of whole messages
  resilient_consensus_critic/_TR return the aggregated estimates (B,1), output layer unchanged (:168-206)
                                 With mixing="nnm", every consensus step first replaces each received message by the
                                 mean of its n - H nearest (nearest-neighbour mixing, rcmarl_nnm_mix); with
                                 mixing="bucket" or ("bucket", s) it keeps its own message and replaces the others by
                                 the means of random buckets of s (randomized bucketing, rcmarl_bucket_mix); with
                                 momentum=beta it replaces slot k's message by its net plus the moving average of
                                 slot k's update against its net (per-neighbour momentum, rcmarl_momentum_mix);
                                 with clipping="arc" it then pulls the k_clip messages furthest from its own in to
                                 the distance of the next (adaptive robust clipping, rcmarl_arc_clip), before mixing
  *_update_team             projection step on the output layer only (:60-84)
  actor_update              one Keras-Adam step weighted by the team TD error (:86-101)
Tensors may be NumPy arrays, torch tensors or facade Tensors; they are moved to the GPU.  Calling these methods one
by one is the compatibility path; training.train_agents.train_RPBCAC drives the same kernels fused over all agents."""
import torch

import tensorflow
from tensorflow import keras
from tensorflow.keras import Tensor
from rcmarl import _lib as L
from rcmarl import agent_ops as A
from rcmarl import nets, ops


class RPBCAC_agent():
    def __init__(self, actor, critic, team_reward, slow_lr, fast_lr, gamma=0.95, H=0, aggregation="clip", mixing=None,
                 momentum=None, clipping=None):
        self.actor = actor
        self.critic = critic
        self.TR = team_reward
        self.gamma = gamma
        self.H = H
        # resilient aggregation rule of every consensus step: "clip" (the reference's), "trim" or "wmsr"
        # (include/rcmarl.h, rcmarl_agg_rule), or a distance-based rule over whole messages: "krum", "mkrum", "scclip"
        # or "gmed" (rcmarl_vector_rule), the spectral rule "dnc" (divide-and-conquer, rcmarl_dnc_aggregate), or the
        # exact subset-selection rules "mda" and "smea" (rcmarl_subset_aggregate), or the iterative outlier scissor "ios"
        # (rcmarl_ios_aggregate)
        if not (L.is_vector_rule(aggregation) or L.is_spectral_rule(aggregation) or L.is_subset_rule(aggregation)
                or L.is_filter_rule(aggregation)):
            L.agg_rule(aggregation)
        self.aggregation = aggregation
        # pre-aggregation mixing of the received messages: None, "nnm", "bucket" or ("bucket", s) (rcmarl_mixing_rule)
        if mixing is not None:
            L.check_mixing(mixing, 0, 1)
        self.mixing = L.mixing_entry(mixing)
        # bucketing draws its permutations from Philox keyed by the facade seed of tf.random.set_seed at construction,
        # with receiver 0 and epoch 0; the round is a per-net count of hidden consensus calls (0 critic, 1 team reward)
        self._bucket_seed = tensorflow.random.seed
        self._consensus_calls = [0, 0]
        # per-neighbour momentum at beta (rcmarl_momentum_mix), or None.  Per net (0 critic, 1 team reward): the state M
        # [n_in, P], created at the first hidden consensus call, and the momentum rows of the last hidden call, which
        # the estimate consensus reuses.  The reference c of a step is the net at its hidden call: the net at the end
        # of the previous consensus round (at construction, for the first).
        if momentum is not None:
            momentum = L.check_momentum(momentum)
            if self.mixing is not None:
                raise L.RcmarlError(f"momentum and mixing {self.mixing!r} together: at most one pre-aggregation step")
        self.momentum = momentum
        # adaptive robust clipping of the stacked rows (rcmarl_arc_clip) after the momentum step, before mixing: None
        # or "arc"
        self.clipping = L.check_clipping(clipping)
        self._momentum_M = [None, None]
        self._momentum_rows = [None, None]
        self.n_actions = self.actor.output_shape[1]
        self.fast_lr = fast_lr
        self.slow_lr = slow_lr
        self.n_agents = critic.n_agents
        self.adam = A.AdamState(slow_lr)                               # :38 Adam(learning_rate=slow_lr)
        self.critic_features = keras.Model(self.critic.inputs, self.critic.layers[-2].output)   # :39
        self.TR_features = keras.Model(self.TR.inputs, self.TR.layers[-2].output)               # :40

    # ------------------------------------------------------------------ aggregation (:42-58)
    def _resilient_aggregation(self, values_innodes):
        v = ops.dev_f32(values_innodes)
        shape = v.shape[1:]
        v = self._mixed(self._clipped(v.reshape(v.shape[0], -1).contiguous()), net=0, round=0)
        if self._whole_messages():                # the rows as whole vectors: out = sum_k w_k v_k
            out = self._with_aggregate(v)[-1]
        elif L.agg_rule(self.aggregation) == L.AGG_CLIP:
            out = ops.clip_mean(v, self.H)
        else:                         # the other rules: one consensus job over all P coordinates of the n rows
            L.check_aggregation(self.aggregation, self.H, v.shape[0])
            out = torch.empty(v.shape[1], dtype=torch.float32, device=v.device)
            ops.consensus_hidden([ops.consensus_job(out, v, v.shape[1], v.shape[1], list(range(v.shape[0])), self.H,
                                                    self.aggregation)])
        return Tensor(out.reshape(shape))

    def _mixed(self, stack, net, round):
        """[n, P] device stack (own = row 0) -> its n nearest-neighbour mixed rows, or its 1 + ceil((n - 1) / s) rows
        bucketed with the draws of (net, round), if the agent mixes; else the stack."""
        if self.mixing is None:
            return stack
        n, P = stack.shape
        L.check_mixing(self.mixing, self.H, n)
        if L.is_bucket_mixing(self.mixing):
            out = torch.empty(L.mixed_rows(self.mixing, n), P, dtype=stack.dtype, device=stack.device)
            ops.bucket_mix([ops.bucket_job(out, stack, P, P, list(range(n)), self.mixing[1], seed=self._bucket_seed,
                                           receiver=0, net=net, round=round & 0xFFFFFFFF, epoch=0)])
            return out
        out = torch.empty_like(stack)
        ops.nnm_mix([ops.vector_job(out, stack, P, P, list(range(n)), self.H, L.MIX_NNM)])
        return out

    def _clipped(self, stack):
        """[n, P] device stack (own = row 0) -> its n rows clipped by ARC at H if the agent clips; else the stack."""
        if self.clipping is None:
            return stack
        n, P = stack.shape
        if not (1 <= n <= L.MAX_NEIGHBOURS and 0 <= self.H < n):
            raise L.RcmarlError(f"clipping 'arc' with H={self.H} needs 0 <= H < n_in (n_in={n}, at most "
                                f"{L.MAX_NEIGHBOURS})")
        out = torch.empty_like(stack)
        ops.arc_clip([ops.vector_job(out, stack, P, P, list(range(n)), self.H, L.MIX_ARC)])
        return out

    def _momentum_step(self, stack, ref, net):
        """[n, P] device stack (own = row 0) -> its n momentum rows against the reference net `ref`, one momentum step
        of net `net` (the first step of each net starts its state)."""
        n, P = stack.shape
        M = self._momentum_M[net]
        first = M is None
        if first:
            M = self._momentum_M[net] = torch.empty_like(stack)
        elif M.shape != stack.shape:
            raise L.RcmarlError(f"momentum keeps one state per slot: this agent's net {net} has heard {M.shape[0]} "
                                f"messages of {M.shape[1]} parameters per round, now {n} of {P}")
        out = torch.empty_like(stack)
        ops.momentum_mix([ops.momentum_job(out, stack, P, P, list(range(n)), ref, M, P, self.momentum, first)])
        self._momentum_rows[net] = out
        return out

    def _whole_messages(self):
        """True if the rule aggregates whole messages (a distance-based rule, dnc, mda, smea or ios)."""
        return (L.is_vector_rule(self.aggregation) or L.is_spectral_rule(self.aggregation)
                or L.is_subset_rule(self.aggregation) or L.is_filter_rule(self.aggregation))

    def _with_aggregate(self, stack):
        """[n, P] device stack (own = row 0) -> [n + 1, P] whose last row is the aggregate of the distance-based, dnc,
        mda, smea or ios rule."""
        n, P = stack.shape
        out = torch.cat([stack, torch.empty(1, P, dtype=stack.dtype, device=stack.device)])
        if L.is_spectral_rule(self.aggregation):
            L.check_spectral_rule(self.H, n)
            ops.dnc_aggregate([ops.vector_job(out[n], out, P, P, list(range(n)), self.H, L.SPECTRAL_DNC)])
        elif L.is_subset_rule(self.aggregation):
            L.check_subset_rule(self.H, n)
            ops.subset_aggregate([ops.vector_job(out[n], out, P, P, list(range(n)), self.H,
                                                 L.SUBSET_RULES[self.aggregation])])
        elif L.is_filter_rule(self.aggregation):
            L.check_filter_rule(self.H, n)
            ops.ios_aggregate([ops.vector_job(out[n], out, P, P, list(range(n)), self.H, L.FILTER_IOS)])
        else:
            L.check_vector_rule(self.aggregation, self.H, n)
            ops.vector_aggregate([ops.vector_job(out[n], out, P, P, list(range(n)), self.H, self.aggregation)])
        return out

    def _consensus_inputs(self, stack, net, round):
        """(message stack, in_nodes, H, rule) of the hidden and estimate consensus over the stacked messages.  A
        distance-based, dnc, mda, smea or ios rule's aggregate becomes the single in-node under clip, which returns it
        exactly, as in Trainer.  An agent that clips does so first, then an agent that mixes does so (a bucketing agent with the draws
        of (net, round))."""
        stack = self._mixed(self._clipped(stack), net, round)
        if self._whole_messages():
            return self._with_aggregate(stack), [stack.shape[0]], 0, "clip"
        return stack, list(range(stack.shape[0])), self.H, self.aggregation

    # ------------------------------------------------------------------ projection step (:60-84)
    def _team(self, model, x, agg):
        rows, kind, xf = A.rows_for(x, self.n_agents)
        B, n = xf.shape[0], model.n_params
        sums = torch.empty(22, dtype=torch.float32, device=xf.device)
        ops.team(rows, [ops.team_job(model.flat, kind, sums=sums, agg_in=A.col(agg))])
        ops.sgd_apply([ops.sgd_job(model.flat, model.flat, sums, n, -1.0 / B, first=n - 21)])

    def critic_update_team(self, s, critic_agg):
        self._team(self.critic, s, critic_agg)

    def TR_update_team(self, sa, TR_agg):
        self._team(self.TR, sa, TR_agg)

    # ------------------------------------------------------------------ actor (:86-101)
    def actor_update(self, s, ns, sa, a_local, pretrain=False):
        NA, g = self.n_agents, float(self.gamma)
        r_team = A.net_values(self.TR.flat, sa, NA)
        nV = A.net_values(self.critic.flat, ns, NA, scale=g, add=r_team)          # r_team + gamma*V(ns)
        delta = A.net_values(self.critic.flat, s, NA, scale=-1.0, add=nV)         # ... - V(s)
        return A.actor_step(self.actor.flat, self.adam, s, a_local, delta, NA)

    # ------------------------------------------------------------------ local updates (:103-140)
    def critic_update_local(self, s, ns, r_local):
        NA = self.n_agents
        target = A.net_values(self.critic.flat, ns, NA, scale=float(self.gamma), add=A.col(r_local))   # :114-115
        msg, loss = A.fit_fullbatch(self.critic.flat, s, target, NA, self.fast_lr, 5)
        return A.DeviceWeights(msg, self.critic.d_in, 1), loss

    def TR_update_local(self, sa, r_local):
        msg, loss = A.fit_fullbatch(self.TR.flat, sa, A.col(r_local), self.n_agents, self.fast_lr, 5)
        return A.DeviceWeights(msg, self.TR.d_in, 1), loss

    # ------------------------------------------------------------------ hidden-layer consensus (:142-166)
    def _hidden(self, model, msgs_innodes, net):
        dev = model.flat.device
        round = self._consensus_calls[net]
        self._consensus_calls[net] += 1
        stack = torch.stack([A.as_flat(m, dev, model.d_in_k) for m in msgs_innodes])
        if self.momentum is not None:                 # against the net before this round's consensus overwrites it
            stack = self._momentum_step(stack, model.flat, net)
        stack, nodes, H, rule = self._consensus_inputs(stack, net, round)
        ops.consensus_hidden([ops.consensus_job(model.flat, stack, stack.shape[1], nets.n_hidden_params(model.d_in_k),
                                                nodes, H, rule)])

    def resilient_consensus_critic_hidden(self, critic_weights_innodes):
        self._hidden(self.critic, critic_weights_innodes, 0)

    def resilient_consensus_TR_hidden(self, TR_weights_innodes):
        self._hidden(self.TR, TR_weights_innodes, 1)

    # ------------------------------------------------------------------ estimate consensus (:168-206)
    def _estimates(self, model, x, msgs_innodes, net):
        # the round of the last hidden consensus of this net: both see the same buckets, as in one Trainer epoch
        rows, kind, xf = A.rows_for(x, self.n_agents)
        dev = xf.device
        if self.momentum is None:
            stack = torch.stack([A.as_flat(m, dev, model.d_in_k) for m in msgs_innodes])
        elif self._momentum_rows[net] is None:
            raise L.RcmarlError("an agent with momentum takes its momentum step at the hidden consensus call: call "
                                "resilient_consensus_*_hidden first")
        else:                                         # the momentum rows of this round's hidden call
            stack = self._momentum_rows[net]
        stack, nodes, H, rule = self._consensus_inputs(stack, net, max(self._consensus_calls[net] - 1, 0))
        agg = torch.empty(xf.shape[0], dtype=torch.float32, device=dev)
        ops.team(rows, [ops.team_job(model.flat, kind, stack, stack.shape[1], nodes, H, agg_out=agg, rule=rule)])
        return Tensor(agg.reshape(-1, 1))

    def resilient_consensus_critic(self, s, critic_weights_innodes):
        return self._estimates(self.critic, s, critic_weights_innodes, 0)

    def resilient_consensus_TR(self, sa, TR_weights_innodes):
        return self._estimates(self.TR, sa, TR_weights_innodes, 1)

    # ------------------------------------------------------------------ acting (:208-219)
    def get_action(self, state, mu=0.1):
        action_prob = self.actor.predict(state).ravel()
        self.action = A.sample_actions(action_prob, self.n_actions, mu)
        return self.action

    def get_parameters(self):
        return [self.actor.get_weights(), self.critic.get_weights(), self.TR.get_weights()]
