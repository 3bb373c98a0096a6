"""train_RPBCAC with the reference's signature and return values (training/train_agents.py:15-184 of
mfigura/Resilient-consensus-based-MARL), executed by the batched device engine (rcmarl.trainer.Trainer):

  * the episodes of a fixed-policy block (n_ep_fixed x max_ep_len steps, :46-80) for ALL environments are one
    rollout kernel launch; there is no per-step host loop;
  * the update round (:86-163) is fused over all agents (Phase I local fits, Phase II resilient consensus +
    projection, Phase III actor steps, Phase IV buffer trim);
  * `env.n_envs` (environments.grid_world.Grid_World(..., n_envs=N) or RCMARL_N_ENVS) independent environments
    share the agents (SURVEY Appendix C); logged returns are means over environments; n_envs == 1 is the reference.

Same printed line per episode, same `sim_data` columns, `weights` as a 1-D object array so that the unchanged
main.py:120 `np.save` works with NumPy >= 1.24."""
import numpy as np
import pandas as pd

from rcmarl.trainer import Trainer

'''
This file contains a function for training consensus AC agents in gym environments. It is designed for batch updates.
'''


def _dist_info():
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except Exception:
        pass
    return 0, 1


def build_trainer(env, agents, args, exp_buffer=None, **overrides):
    """Reference objects (env, agents, args) -> device engine.  Agent weights / Adam slots are read once here and
    written back by `sync_agents` after training."""
    labels = list(args['agent_label'])
    weights = [ag.get_parameters() for ag in agents]
    slow_lr = [float(getattr(ag, 'slow_lr', args.get('slow_lr', 0.01))) for ag in agents]
    # per-agent hyper-parameters, as the reference stores them (agents/resilient_CAC_agents.py:28-36)
    fast = [float(getattr(ag, 'fast_lr', args.get('fast_lr', 0.01))) for ag in agents]
    H = [int(getattr(ag, 'H', 0)) for ag in agents]
    aggregation = [getattr(ag, 'aggregation', 'clip') for ag in agents]
    attack = [getattr(ag, 'attack', None) for ag in agents]                # Byzantine_CAC_agent
    mixing = [getattr(ag, 'mixing', None) for ag in agents]                # RPBCAC_agent: None, "nnm" or ("bucket", s)
    momentum = [getattr(ag, 'momentum', None) for ag in agents]            # RPBCAC_agent: None or beta
    clipping = [getattr(ag, 'clipping', None) for ag in agents]            # RPBCAC_agent: None or "arc"
    adam = [(ag.adam.m, ag.adam.v, ag.adam.t) if getattr(ag, 'adam', None) is not None and ag.adam.m is not None else None
            for ag in agents]
    rank, world = _dist_info()
    # Grid_World options of the reference (grid_world.py:21-45): state scaling and fixed / random resets
    scaling = bool(np.any(np.asarray(getattr(env, 'std_state', 1)) != 1) or np.any(np.asarray(getattr(env, 'mean_state', 0)) != 0))
    fixed0 = None if getattr(env, 'randomize_state', True) else env.initial_state
    kw = dict(scaling=scaling, fixed_initial_state=fixed0, labels=labels, in_nodes=args['in_nodes'], weights=weights, desired=env.desired_state,
              n_envs=getattr(env, 'n_envs', 1), nrow=env.nrow, ncol=env.ncol, gamma=args['gamma'], H=H, fast_lr=fast, slow_lr=slow_lr, max_ep_len=args['max_ep_len'],
              n_ep_fixed=args['n_ep_fixed'], n_epochs=args['n_epochs'], buffer_size=args['buffer_size'],
              common_reward=bool(args['common_reward']), seed=int(args.get('random_seed', 0)), adam_state=adam,
              rank=rank, world=world, aggregation=aggregation, attack=attack, mixing=mixing,
              momentum=momentum, clipping=clipping)
    kw.update(overrides)
    tr = Trainer(**kw)
    if exp_buffer:                                                             # :36-40
        tr.load_rows(exp_buffer[0], exp_buffer[1], exp_buffer[2], exp_buffer[3])
    return tr


def sync_agents(tr, agents):
    """Write the trained parameters / Adam slots back into the agent objects."""
    for i, ag in enumerate(agents):
        w = tr.get_weights(i)
        ag.actor.set_weights(w[0])
        ag.critic.set_weights(w[1])
        ag.TR.set_weights(w[2])
        if len(w) > 3:
            ag.critic_local_weights = w[3]
        if getattr(ag, 'adam', None) is not None:
            ag.adam.m, ag.adam.v, ag.adam.t = tr.adam_m[i].clone(), tr.adam_v[i].clone(), tr.adam_t[i]


def train_RPBCAC(env, agents, args, exp_buffer=None, verbose=True):
    '''
    FUNCTION train_RPBCAC() - training a mixed cooperative and adversarial network of consensus AC agents including
    RPBCAC agents (same contract as the reference).
    ARGUMENTS: gym environment, list of agents, user-defined parameters for the simulation
    RETURNS: (weights, sim_data)
    '''
    paths = []
    n_agents = env.n_agents
    labels = args['agent_label']
    n_coop = labels.count('Cooperative')
    coop = [i for i in range(n_agents) if labels[i] == 'Cooperative']
    adv = [i for i in range(n_agents) if labels[i] != 'Cooperative']
    n_episodes, n_ep_fixed = args['n_episodes'], args['n_ep_fixed']
    tr = build_trainer(env, agents, args, exp_buffer)
    zeros = np.zeros(n_agents)
    t = 0
    while t < n_episodes:
        n_ep = min(n_ep_fixed, n_episodes - t)
        est, ret = tr.rollout_block(n_ep)                                      # :46-80 for every environment
        losses = tr.update_round() if n_ep == n_ep_fixed else None             # :86 (i == n_ep_fixed-1)
        for e in range(n_ep):
            last = losses is not None and e == n_ep - 1
            critic_loss = losses['critic_loss'] if last else zeros
            TR_loss = losses['TR_loss'] if last else zeros
            actor_loss = losses['actor_loss'] if last else zeros
            est_returns = [est[e, i] for i in coop]
            mean_true_returns = float(np.sum(ret[e, coop]) / n_coop) if n_coop else 0
            mean_true_returns_adv = float(np.sum(ret[e, adv]) / (n_agents - n_coop)) if adv else 0
            if verbose:
                print('| Episode: {} | Est. returns: {} | Returns: {} | Average critic loss: {} | Average TR loss: {} | Average actor loss: {} '.format(t + e, est_returns, mean_true_returns, critic_loss, TR_loss, actor_loss))
            paths.append({"True_team_returns": mean_true_returns,
                          "True_adv_returns": mean_true_returns_adv,
                          "Estimated_team_returns": np.mean(est_returns) if est_returns else np.nan})
        t += n_ep
    sim_data = pd.DataFrame.from_dict(paths)
    sync_agents(tr, agents)
    weights = np.empty(n_agents, dtype=object)                                 # np.save-able (SURVEY 5)
    for i, agent in enumerate(agents):
        weights[i] = agent.get_parameters()
    train_RPBCAC.last_trainer = tr
    return weights, sim_data
