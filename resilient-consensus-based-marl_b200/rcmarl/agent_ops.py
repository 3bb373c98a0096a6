"""Per-agent building blocks shared by the reference-shaped Agent classes (agents/*.py in this tree).
Every function takes device tensors and launches librcmarl.so kernels through rcmarl.ops; nothing here
computes on the host.  The fused multi-agent schedule lives in rcmarl.trainer."""
import numpy as np
import torch

from . import _lib as L
from . import nets, ops


class DeviceWeights(list):
    """A transmitted message: behaves like the reference's list of six ndarrays (training/train_agents.py:120-121,
    129-130) and carries the packed device copy the kernels read."""

    def __init__(self, flat, d_in, n_out):
        d_in_k = (flat.numel() - (L.HIDDEN + L.HIDDEN * L.HIDDEN + L.HIDDEN + L.HIDDEN * n_out + n_out)) // L.HIDDEN
        super().__init__(nets.unpack_padded(flat.detach().cpu().numpy(), d_in, d_in_k, n_out))
        self.flat, self.d_in, self.n_out = flat, d_in, n_out


def as_flat(msg, device, d_in_k=None):
    if hasattr(msg, "flat"):
        return msg.flat
    if d_in_k is None:
        return torch.as_tensor(nets.pack(msg)).to(device)
    return torch.as_tensor(nets.pack_padded(msg, d_in_k)).to(device)


def rows_for(x, n_agents):
    """(B, n_agents, f) tensor -> (rows struct, input kind, flat device view).  f == 3 feeds IN_SA, f == 2 is handed
    over through the `ns` slot (contiguous [B][2*n_agents])."""
    x = ops.dev_f32(x)
    B = x.shape[0]
    x = x.reshape(B, -1)
    nk = nets.kernel_agents(n_agents)                       # kernel instantiation; extra agent slots stay zero
    if x.shape[1] == 3 * n_agents:
        x = nets.pad_agent_slots(x, n_agents, nk)
        return ops.make_rows(x, None, None, nk), L.IN_SA, x
    if x.shape[1] == 2 * n_agents:
        x = nets.pad_agent_slots(x, n_agents, nk)
        return ops.make_rows(None, x, None, nk), L.IN_NS, x
    raise ValueError(f"unexpected feature count {x.shape[1]} for {n_agents} agents")


def col(y):
    """(B,1) / (B,) host or device -> contiguous float32 device vector [B]."""
    return ops.dev_f32(y).reshape(-1).contiguous()


def net_values(w, x, n_agents, scale=1.0, add=None, add_scale=1.0):
    rows, kind, _x = rows_for(x, n_agents)
    out = torch.empty(_x.shape[0], dtype=torch.float32, device=_x.device)
    ops.values(rows, [ops.value_job(out, [(w, kind, scale)], add=add, add_scale=add_scale)])
    return out


def fit_fullbatch(w, x, target, n_agents, lr, epochs=5):
    """model.fit(x, y, batch_size=B, epochs=5) with SGD on a COPY of the weights
    (agents/resilient_CAC_agents.py:113-122,133-140).  Returns (updated copy, history['loss'][0])."""
    rows, kind, xf = rows_for(x, n_agents)
    B, n = xf.shape[0], w.numel()
    msg = torch.empty_like(w)
    sums = torch.empty(n + 1, dtype=torch.float32, device=w.device)
    loss = torch.zeros(1, dtype=torch.float32, device=w.device)
    for e in range(epochs):
        src = w if e == 0 else msg
        ops.grad(rows, [ops.grad_job(src, target, sums, kind)], L.LOSS_MSE)
        ops.sgd_apply([ops.sgd_job(msg, src, sums, n, lr * 2.0 / B, loss_out=loss if e == 0 else None, loss_coef=1.0 / B)])
    return msg, float(loss.item())


def fit_minibatch(w, x, target, n_agents, lr, epochs, mb_times, perms, n_envs=1):
    """model.fit(x, y, epochs=10, batch_size=32) with shuffling, IN PLACE
    (agents/adversarial_CAC_agents.py:133,150,163,239,251).  perms: int32 device tensor [epochs, T] of time-row
    permutations; a mini-batch is mb_times time rows x n_envs environments (SURVEY Appendix C)."""
    rows, kind, xf = rows_for(x, n_agents)
    B, n = xf.shape[0], w.numel()
    rows.n_envs = n_envs
    rows.time_idx = perms.data_ptr()
    sums = torch.empty(n + 1, dtype=torch.float32, device=w.device)
    loss = torch.zeros(1, dtype=torch.float32, device=w.device)
    ops.minibatch_steps(rows, [ops.grad_job(w, target, sums, kind, time_idx=perms)],
                        [ops.sgd_job(w, w, sums, n, 0.0, loss_out=loss, loss_coef=1.0 / B, loss_accumulate=1)],
                        epochs, B // n_envs, mb_times, [lr])
    return float(loss.item())


class AdamState:
    """Keras Adam slots of one actor (persist for the life of the agent, SURVEY Appendix A.5)."""

    def __init__(self, lr):
        self.lr, self.t, self.m, self.v = float(lr), 0, None, None

    def ensure(self, like):
        if self.m is None:
            self.m, self.v = torch.zeros_like(like), torch.zeros_like(like)


def _sa_with_action(s, a_local, n_agents):
    """Rows for the CE kernel: it reads the action from sa[row][3*agent+2]; the per-agent API passes the agent's
    own action column separately, so it is placed in slot 0 of a temporary sa layout (pure data movement)."""
    s = ops.dev_f32(s)
    B = s.shape[0]
    sa = torch.zeros(B, nets.kernel_agents(n_agents), 3, dtype=torch.float32, device=s.device)
    sa[:, :n_agents, :2] = s.reshape(B, n_agents, 2)
    sa[:, 0, 2] = col(a_local)
    return sa.reshape(B, -1)


def actor_step(actor_w, adam, s, a_local, delta, n_agents):
    """actor.train_on_batch(s, a_local, sample_weight=delta) (agents/resilient_CAC_agents.py:99)."""
    sa = _sa_with_action(s, a_local, n_agents)
    B, n = sa.shape[0], actor_w.numel()
    rows = ops.make_rows(sa, None, None, nets.kernel_agents(n_agents))
    adam.ensure(actor_w)
    sums = torch.empty(n + 1, dtype=torch.float32, device=actor_w.device)
    loss = torch.zeros(1, dtype=torch.float32, device=actor_w.device)
    adam.t += 1
    ops.grad(rows, [ops.grad_job(actor_w, delta, sums, L.IN_S, action_agent=0)], L.LOSS_CE)
    ops.adam_apply([ops.adam_job(actor_w, adam.m, adam.v, sums, n, 1.0 / B, ops.keras_adam_lr_t(adam.lr, adam.t),
                                 loss_out=loss, loss_coef=1.0 / B)])
    return float(loss.item())


def actor_fit_minibatch(actor_w, adam, s, a_local, delta, n_agents, mb_times, perm, n_envs=1):
    """actor.fit(s, a_local, sample_weight=TD, batch_size=200, epochs=1) (agents/adversarial_CAC_agents.py:41,116,224)."""
    sa = _sa_with_action(s, a_local, n_agents)
    B, n = sa.shape[0], actor_w.numel()
    rows = ops.make_rows(sa, None, None, nets.kernel_agents(n_agents), time_idx=perm, n_envs=n_envs)
    adam.ensure(actor_w)
    sums = torch.empty(n + 1, dtype=torch.float32, device=actor_w.device)
    loss = torch.zeros(1, dtype=torch.float32, device=actor_w.device)
    adam.t += ops.adam_minibatch_steps(
        rows, [ops.grad_job(actor_w, delta, sums, L.IN_S, action_agent=0, time_idx=perm)],
        [ops.adam_job(actor_w, adam.m, adam.v, sums, n, 0.0, 0.0, loss_out=loss, loss_coef=1.0 / B, loss_accumulate=1)],
        B // n_envs, mb_times, [adam.lr], [adam.t])
    return float(loss.item())


_perm_rng = np.random.RandomState(0)


def draw_perms(n, T, device, source=None):
    """n permutations of range(T) as an int32 device tensor [n, T].  `source` (callable T -> permutation) lets
    tests inject the shuffles; otherwise a module-level NumPy stream is used (Keras' shuffle RNG is private too)."""
    ps = [np.asarray(source(T) if source is not None else _perm_rng.permutation(T), np.int32) for _ in range(n)]
    return torch.as_tensor(np.stack(ps)).to(device)


def sample_actions(probs, n_actions, mu):
    """get_action (agents/resilient_CAC_agents.py:208-219) for one row, drawing from NumPy's global RNG in the
    reference's order (choice(n); choice(n, p); choice([a_pol, a_rand], p=[1-mu, mu]))."""
    random_action = np.random.choice(n_actions)
    p = np.asarray(probs, np.float64).ravel()
    action_from_policy = np.random.choice(n_actions, p=p / p.sum())
    return np.random.choice([action_from_policy, random_action], p=[1 - mu, mu])
