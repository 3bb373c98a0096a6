"""RPBCAC_agent with the reference's API (agents/resilient_CAC_agents.py:5-223 of
mfigura/Resilient-consensus-based-MARL), executed by the sm_90a kernels of librcmarl.so.

Same constructor and method names, argument meaning and mutation conventions as the reference (SURVEY.md 8b):
  *_update_local            return (message copy, loss) and leave the agent's own networks untouched (:113,120)
  resilient_consensus_*_hidden   overwrite the hidden layers with the clipped mean of the neighbours' (:142-166), or
                                 their trimmed / W-MSR mean with aggregation="trim" / "wmsr"
  resilient_consensus_critic/_TR return the aggregated estimates (B,1), output layer unchanged (:168-206)
  *_update_team             projection step on the output layer only (:60-84)
  actor_update              one Keras-Adam step weighted by the team TD error (:86-101)
Tensors may be NumPy arrays, torch tensors or facade Tensors; they are moved to the GPU.  Calling these methods one
by one is the compatibility path; training.train_agents.train_RPBCAC drives the same kernels fused over all agents."""
import torch

from tensorflow import keras
from tensorflow.keras import Tensor
from rcmarl import _lib as L
from rcmarl import agent_ops as A
from rcmarl import nets, ops


class RPBCAC_agent():
    def __init__(self, actor, critic, team_reward, slow_lr, fast_lr, gamma=0.95, H=0, aggregation="clip"):
        self.actor = actor
        self.critic = critic
        self.TR = team_reward
        self.gamma = gamma
        self.H = H
        # resilient aggregation rule of every consensus step: "clip" (the reference's), "trim" or "wmsr"
        # (include/rcmarl.h, rcmarl_agg_rule)
        L.agg_rule(aggregation)
        self.aggregation = aggregation
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
        v = v.reshape(v.shape[0], -1)
        if L.agg_rule(self.aggregation) == L.AGG_CLIP:
            out = ops.clip_mean(v, self.H)
        else:                         # the other rules: one consensus job over all P coordinates of the n rows
            L.check_aggregation(self.aggregation, self.H, v.shape[0])
            out = torch.empty(v.shape[1], dtype=torch.float32, device=v.device)
            ops.consensus_hidden([ops.consensus_job(out, v, v.shape[1], v.shape[1], list(range(v.shape[0])), self.H,
                                                    self.aggregation)])
        return Tensor(out.reshape(shape))

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
    def _hidden(self, model, msgs_innodes):
        dev = model.flat.device
        stack = torch.stack([A.as_flat(m, dev, model.d_in_k) for m in msgs_innodes])
        ops.consensus_hidden([ops.consensus_job(model.flat, stack, stack.shape[1], nets.n_hidden_params(model.d_in_k),
                                                list(range(len(msgs_innodes))), self.H, self.aggregation)])

    def resilient_consensus_critic_hidden(self, critic_weights_innodes):
        self._hidden(self.critic, critic_weights_innodes)

    def resilient_consensus_TR_hidden(self, TR_weights_innodes):
        self._hidden(self.TR, TR_weights_innodes)

    # ------------------------------------------------------------------ estimate consensus (:168-206)
    def _estimates(self, model, x, msgs_innodes):
        rows, kind, xf = A.rows_for(x, self.n_agents)
        dev = xf.device
        stack = torch.stack([A.as_flat(m, dev, model.d_in_k) for m in msgs_innodes])
        agg = torch.empty(xf.shape[0], dtype=torch.float32, device=dev)
        ops.team(rows, [ops.team_job(model.flat, kind, stack, stack.shape[1], list(range(len(msgs_innodes))), self.H,
                                     agg_out=agg, rule=self.aggregation)])
        return Tensor(agg.reshape(-1, 1))

    def resilient_consensus_critic(self, s, critic_weights_innodes):
        return self._estimates(self.critic, s, critic_weights_innodes)

    def resilient_consensus_TR(self, sa, TR_weights_innodes):
        return self._estimates(self.TR, sa, TR_weights_innodes)

    # ------------------------------------------------------------------ acting (:208-219)
    def get_action(self, state, mu=0.1):
        action_prob = self.actor.predict(state).ravel()
        self.action = A.sample_actions(action_prob, self.n_actions, mu)
        return self.action

    def get_parameters(self):
        return [self.actor.get_weights(), self.critic.get_weights(), self.TR.get_weights()]
