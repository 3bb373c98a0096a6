"""Adversarial agents with the reference's API (agents/adversarial_CAC_agents.py of
mfigura/Resilient-consensus-based-MARL) on the sm_90a kernels of librcmarl.so.

  Faulty_CAC_agent     :5-72    transmits fixed critic / TR parameters, trains only its actor
  Malicious_CAC_agent  :74-182  private local critic + compromised critic / TR trained on -r_coop and transmitted
  Greedy_CAC_agent     :184-275 trains critic / TR on its own reward and transmits them
  Byzantine_CAC_agent  (not in the reference) learns like Faulty; sends each cooperative receiver its own crafted message
Mini-batch fits use Keras defaults (batch_size rows shuffled per epoch, SURVEY Appendix A.3).  The shuffle stream is
private (like TF's); `perm_source` (callable T -> permutation) can be set on an agent to inject it."""
import numpy as np

from rcmarl import agent_ops as A


class _AdversaryBase():
    perm_source = None
    n_envs = 1                                      # Appendix C: a mini-batch is batch_size time rows x n_envs

    def _init_common(self, actor, critic, team_reward, slow_lr, gamma):
        self.actor = actor
        self.critic = critic
        self.TR = team_reward
        self.gamma = gamma
        self.n_actions = self.actor.output_shape[1]
        self.n_agents = critic.n_agents
        self.slow_lr = slow_lr
        self.adam = A.AdamState(slow_lr)

    def _perms(self, n, B, device):
        return A.draw_perms(n, B // self.n_envs, device, self.perm_source)

    def _td_error(self, critic_w, s, ns, r_local):
        NA, g = self.n_agents, float(self.gamma)
        nV = A.net_values(critic_w, ns, NA, scale=g, add=A.col(r_local))          # r + gamma*V(ns)
        return A.net_values(critic_w, s, NA, scale=-1.0, add=nV)                   # ... - V(s)

    def _actor_fit(self, critic_w, s, ns, r_local, a_local):
        delta = self._td_error(critic_w, s, ns, r_local)
        perm = self._perms(1, delta.numel(), delta.device)[0]
        return A.actor_fit_minibatch(self.actor.flat, self.adam, s, a_local, delta, self.n_agents, 200, perm, self.n_envs)

    def _critic_fit(self, w, s, ns, r, target_w=None):
        """TD target from `target_w` (default: w itself, before the fit), then 10 epochs x batch 32 in place."""
        NA = self.n_agents
        target = A.net_values(w if target_w is None else target_w, ns, NA, scale=float(self.gamma), add=A.col(r))
        return A.fit_minibatch(w, s, target, NA, self.fast_lr, 10, 32, self._perms(10, target.numel(), w.device), self.n_envs)

    def _tr_fit(self, w, sa, r):
        t = A.col(r)
        return A.fit_minibatch(w, sa, t, self.n_agents, self.fast_lr, 10, 32, self._perms(10, t.numel(), w.device), self.n_envs)

    def get_action(self, state, mu=0.1):
        action_prob = self.actor.predict(state).ravel()
        self.action = A.sample_actions(action_prob, self.n_actions, mu)
        return self.action

    def get_parameters(self):
        return [self.actor.get_weights(), self.critic.get_weights(), self.TR.get_weights()]


class Faulty_CAC_agent(_AdversaryBase):
    def __init__(self, actor, critic, team_reward, slow_lr, gamma=0.95):
        self._init_common(actor, critic, team_reward, slow_lr, gamma)

    def actor_update(self, s, ns, r_local, a_local):                               # :28-43
        return self._actor_fit(self.critic.flat, s, ns, r_local, a_local)

    def get_critic_weights(self):                                                   # :45-49
        return A.DeviceWeights(self.critic.flat.clone(), self.critic.d_in, 1)

    def get_TR_weights(self):                                                       # :51-55
        return A.DeviceWeights(self.TR.flat.clone(), self.TR.d_in, 1)


class Byzantine_CAC_agent(Faulty_CAC_agent):
    """Learns like Faulty_CAC_agent; what it transmits is crafted by the training loop for each cooperative receiver
    from that receiver's honest neighbours (`attack` = ("alie", z), ("ipm", eps) or ("gauss", s), threat model at
    rcmarl_attack in include/rcmarl.h; or a min-max / min-sum attack scaled to the receiver's honest spread,
    ("minmax_uv" | "minmax_std" | "minmax_sgn" | "minsum_uv" | "minsum_std" | "minsum_sgn", s) with s >= 0 and s = 1 the
    paper's attack, at rcmarl_adaptive_attack; or a rule-aware attack tuned against the receiver's own rule and H,
    ("tailored_uv" | "tailored_std" | "tailored_sgn", s) with the range multiplier s >= 0, at rcmarl_tailored_attack; or
    the same search against the receiver's whole pipeline -- its mixing step (nnm or bucketing, the latter over shuffles
    of the attacker's own) and then its rule, DnC included -- ("pipeline_uv" | "pipeline_std" | "pipeline_sgn", s), at
    rcmarl_pipeline_attack; or that search run in the momentum rows of a receiver with momentum and inverted through
    its momentum step, ("history_uv" | "history_std" | "history_sgn", s), at rcmarl_history_attack (against a receiver
    without momentum it is the pipeline attack in the same direction); or that history / pipeline search through the
    receiver's adaptive robust clipping as well, ("arc_uv" | "arc_std" | "arc_sgn", s), at rcmarl_history_arc_attack /
    rcmarl_pipeline_arc_attack (against a receiver that does not clip it is the history attack); or that search through
    an mda / smea receiver's exact subset selection as well, ("subset_uv" | "subset_std" | "subset_sgn", s), at
    rcmarl_subset_history_attack / rcmarl_subset_pipeline_attack (against a receiver on any other rule it is the ARC
    attack); or that search through an ios receiver's iterative outlier scissor as well, ("ios_uv" | "ios_std" |
    "ios_sgn", s), at rcmarl_ios_history_attack / rcmarl_ios_pipeline_attack (against a receiver on any other rule it
    is the subset attack); or the dissensus attack that cancels (eps = 1) or reverses (eps > 1) the receiver's honest pull, ("dissensus", eps)
    with eps >= 0, at rcmarl_dissensus_attack; or the mimic attack that copies the honest neighbour furthest along the
    honest messages' principal direction, ("mimic", T0) with T0 the number of power steps, an integer in 0 .. 2^31 - 1,
    after which the direction is frozen, at rcmarl_mimic_attack).
    The reference has no such agent: train_RPBCAC reads `attack` from it, under
    the label "Byzantine".  get_critic_weights / get_TR_weights return the untouched nets, as Faulty's do: an agent
    alone has no view of its receivers' neighbourhoods."""

    def __init__(self, actor, critic, team_reward, slow_lr, gamma=0.95, attack=None):
        super().__init__(actor, critic, team_reward, slow_lr, gamma)
        from rcmarl import _lib
        _lib.check_attack(attack)
        self.attack = (attack[0], float(attack[1]))


class Malicious_CAC_agent(_AdversaryBase):
    def __init__(self, actor, critic, team_reward, slow_lr, fast_lr, gamma=0.95):
        self._init_common(actor, critic, team_reward, slow_lr, gamma)
        self.fast_lr = fast_lr
        self._critic_local = None
        self._critic_local_host = self.critic.get_weights()                         # :99

    # main.py:92 assigns `agent.critic_local_weights = pretrained_weights[node][3]`
    @property
    def critic_local_weights(self):
        if self._critic_local is None:
            return self._critic_local_host
        from rcmarl import nets
        return nets.unpack_padded(self._critic_local.detach().cpu().numpy(), self.critic.d_in, self.critic.d_in_k, 1)

    @critic_local_weights.setter
    def critic_local_weights(self, w):
        self._critic_local_host = [np.asarray(a, np.float32) for a in w]
        self._critic_local = None

    @property
    def critic_local_flat(self):
        if self._critic_local is None:
            import torch
            from rcmarl import nets
            self._critic_local = torch.as_tensor(nets.pack_padded(self._critic_local_host, self.critic.d_in_k)).to(self.critic.flat.device)
        return self._critic_local

    def actor_update(self, s, ns, r_local, a_local):                               # :102-119
        return self._actor_fit(self.critic_local_flat, s, ns, r_local, a_local)

    def critic_update_compromised(self, s, ns, r_compromised):                     # :121-135
        loss = self._critic_fit(self.critic.flat, s, ns, r_compromised)
        return A.DeviceWeights(self.critic.flat.clone(), self.critic.d_in, 1), loss

    def critic_update_local(self, s, ns, r_local):                                 # :137-152
        self._critic_fit(self.critic_local_flat, s, ns, r_local)

    def TR_update_compromised(self, sa, r_compromised):                            # :154-165
        loss = self._tr_fit(self.TR.flat, sa, r_compromised)
        return A.DeviceWeights(self.TR.flat.clone(), self.TR.d_in, 1), loss

    def get_parameters(self):                                                       # :180-182
        return [self.actor.get_weights(), self.critic.get_weights(), self.TR.get_weights(), self.critic_local_weights]


class Greedy_CAC_agent(_AdversaryBase):
    def __init__(self, actor, critic, team_reward, slow_lr, fast_lr, gamma=0.95):
        self._init_common(actor, critic, team_reward, slow_lr, gamma)
        self.fast_lr = fast_lr

    def actor_update(self, s, ns, r_local, a_local):                               # :211-226
        return self._actor_fit(self.critic.flat, s, ns, r_local, a_local)

    def critic_update_local(self, s, ns, r_local):                                 # :228-241
        loss = self._critic_fit(self.critic.flat, s, ns, r_local)
        return A.DeviceWeights(self.critic.flat.clone(), self.critic.d_in, 1), loss

    def TR_update_local(self, sa, r_local):                                        # :243-253
        loss = self._tr_fit(self.TR.flat, sa, r_local)
        return A.DeviceWeights(self.TR.flat.clone(), self.TR.d_in, 1), loss
