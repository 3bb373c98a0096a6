"""CPU ORACLE for the RPBCAC training hot path -- TEST INFRASTRUCTURE ONLY.

This module is a NumPy restatement of the reference algorithm
(mfigura/Resilient-consensus-based-MARL @ f10f8631).  It is *not* part of the
product: only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import it.  The product path
(``resilient-consensus-based-marl_b200/``) never imports anything from
``oracle/`` and fails loudly when its CUDA library is missing.

Parity pinning status
---------------------
* PINNED by the reference's own artefacts: Dense layout / flatten order /
  LeakyReLU slope / state scaling / NumPy RNG draw order, through the logged
  ``Est. returns`` of ``simulation_results/raw_data/*/H=*/seed=*/out.txt``
  (tests/golden/kat_est_returns.npz, tests/test_oracle_kat.py).
* PINNED against the reference sources executed verbatim on a NumPy
  TensorFlow/Keras facade (``oracle/tf_facade``; fixtures in
  tests/golden/ref_on_facade_*.npz made by ``oracle/make_golden.py``):
  control flow of every Agent method, the training schedule, the environment.
* UNPINNED ("parity unpinned"): the Keras-internal arithmetic of ``fit`` /
  ``train_on_batch`` / Adam / loss reductions.  TensorFlow 2.4 is not
  installable here and the reference has no tests; those semantics follow
  SURVEY.md Appendix A ([TF-semantics]) in BOTH the facade and this file.

Every function cites the reference file:line it restates.  All arithmetic is
done in ``dtype`` (float32 to mirror the reference, float64 as a tighter
yardstick for the CUDA kernels).
"""
from __future__ import annotations

import numpy as np

LRELU_SLOPE = 0.1          # main.py:63-65  keras.layers.LeakyReLU(alpha=0.1)
HIDDEN = 20                # main.py:63-64  Dense(20)


# ----------------------------------------------------------------------------
# MLP primitives (main.py:60-82; SURVEY Appendix A.1)
# ----------------------------------------------------------------------------
def lrelu(z):
    return np.where(z > 0, z, z.dtype.type(LRELU_SLOPE) * z)


def lrelu_grad(z):
    # tf.nn.leaky_relu gradient: g where features > 0 else alpha * g
    one = z.dtype.type(1.0)
    return np.where(z > 0, one, z.dtype.type(LRELU_SLOPE))


def cast_weights(w, dtype):
    return [np.asarray(a, dtype=dtype).copy() for a in w]


def flatten_rows(x, dtype):
    """keras.layers.Flatten: row-major over (agent, feature) (main.py:61-62)."""
    x = np.asarray(x, dtype=dtype)
    return x.reshape(x.shape[0], -1)


def mlp_forward(w, x, cache=False):
    """x: (B, d_in) already flattened.  Returns raw last-layer output (logits
    for the actor, value for critic / TR)."""
    W1, b1, W2, b2, W3, b3 = w
    z1 = x @ W1 + b1
    h1 = lrelu(z1)
    z2 = h1 @ W2 + b2
    h2 = lrelu(z2)
    out = h2 @ W3 + b3
    if cache:
        return out, (x, z1, h1, z2, h2)
    return out


def mlp_features(w, x):
    """critic_features / TR_features = model up to layers[-2]
    (agents/resilient_CAC_agents.py:39-40)."""
    W1, b1, W2, b2 = w[:4]
    return lrelu(lrelu(x @ W1 + b1) @ W2 + b2)


def mlp_backward(w, cache_, dout, last_layer_only=False):
    """Gradient of sum(dout * out) w.r.t. the six arrays."""
    W1, b1, W2, b2, W3, b3 = w
    x, z1, h1, z2, h2 = cache_
    gW3 = h2.T @ dout
    gb3 = dout.sum(0)
    if last_layer_only:
        return [np.zeros_like(W1), np.zeros_like(b1), np.zeros_like(W2),
                np.zeros_like(b2), gW3, gb3]
    d2 = (dout @ W3.T) * lrelu_grad(z2)
    gW2 = h1.T @ d2
    gb2 = d2.sum(0)
    d1 = (d2 @ W2.T) * lrelu_grad(z1)
    gW1 = x.T @ d1
    gb1 = d1.sum(0)
    return [gW1, gb1, gW2, gb2, gW3, gb3]


def softmax(logits):
    m = logits.max(axis=1, keepdims=True)
    e = np.exp(logits - m)
    return e / e.sum(axis=1, keepdims=True)


def log_softmax(logits):
    m = logits.max(axis=1, keepdims=True)
    s = logits - m
    return s - np.log(np.exp(s).sum(axis=1, keepdims=True))


# ----------------------------------------------------------------------------
# Keras training semantics (SURVEY Appendix A.2-A.5, [TF-semantics])
# ----------------------------------------------------------------------------
def mse_step(w, x, y, lr, sample_weight=None, last_layer_only=False):
    """One SGD step on Keras MeanSquaredError (SUM_OVER_BATCH_SIZE):
    loss = sum_i w_i * (pred_i - y_i)^2 / B.  Returns (new_w, loss_before)."""
    dt = x.dtype.type
    B = x.shape[0]
    out, cch = mlp_forward(w, x, cache=True)
    err = out - y
    sw = np.ones((B, 1), x.dtype) if sample_weight is None else \
        np.asarray(sample_weight, x.dtype).reshape(B, 1)
    loss = (sw * err * err).sum() / dt(B)
    dout = dt(2.0) * sw * err / dt(B)
    g = mlp_backward(w, cch, dout, last_layer_only=last_layer_only)
    new_w = [a - dt(lr) * ga for a, ga in zip(w, g)]
    if last_layer_only:
        new_w[:4] = [a.copy() for a in w[:4]]
    return new_w, loss


def fit_fullbatch(w, x, y, lr, epochs):
    """model.fit(x, y, batch_size=B, epochs=epochs) with plain SGD
    (agents/resilient_CAC_agents.py:118,136; Appendix A.3).
    Returns (weights after `epochs` steps, history['loss'][0])."""
    loss0 = None
    for e in range(epochs):
        w, loss = mse_step(w, x, y, lr)
        if e == 0:
            loss0 = loss
    return w, loss0


def fit_minibatch(w, x, y, lr, epochs, batch_size, perms):
    """model.fit(x, y, epochs=epochs, batch_size=batch_size) with shuffle=True
    (agents/adversarial_CAC_agents.py:133,150,163,239,251; Appendix A.3).
    perms: (epochs, B) int array -- the per-epoch row permutations (TF's own
    RNG is unreproducible, so they are injected).
    history['loss'][0] = sample-count weighted mean of epoch-0 batch losses."""
    B = x.shape[0]
    loss_acc, cnt = 0.0, 0
    for e in range(epochs):
        p = np.asarray(perms[e])
        for k in range(0, B, batch_size):
            idx = p[k:k + batch_size]
            w, loss = mse_step(w, x[idx], y[idx], lr)
            if e == 0:
                loss_acc += float(loss) * len(idx)
                cnt += len(idx)
    return w, x.dtype.type(loss_acc / cnt)


class KerasAdam:
    """Adam as implemented by TF-2.x Keras (Appendix A.5): epsilon added to
    sqrt(v) without bias correction, lr_t = lr*sqrt(1-b2^t)/(1-b1^t).

    fp32_betas=True: the moment updates take beta1, beta2 as the float32
    constants (0.9f, 0.999f) and 1 - beta as their float32 difference
    (1.f - 0.999f = 0.00099998713, 1.3e-5 below 0.001), as TF does for
    float32 variables and as rcmarl_adam_apply does; lr_t keeps the exact
    constants (ops.keras_adam_lr_t).  The default keeps 1 - 0.999 exact."""

    def __init__(self, lr, beta1=0.9, beta2=0.999, eps=1e-7, fp32_betas=False):
        self.lr, self.b1, self.b2, self.eps = lr, beta1, beta2, eps
        self.fp32_betas = fp32_betas
        self.t = 0
        self.m = None
        self.v = None

    def step(self, w, g):
        dt = w[0].dtype.type
        if self.m is None:
            self.m = [np.zeros_like(a) for a in w]
            self.v = [np.zeros_like(a) for a in w]
        self.t += 1
        lr_t = dt(self.lr * np.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t))
        b1, b2 = self.b1, self.b2
        if self.fp32_betas:                          # 1 - b is then exact in fp64 (Sterbenz)
            b1, b2 = float(np.float32(b1)), float(np.float32(b2))
        out = []
        for i, (a, ga) in enumerate(zip(w, g)):
            self.m[i] = dt(b1) * self.m[i] + dt(1.0 - b1) * ga
            self.v[i] = dt(b2) * self.v[i] + dt(1.0 - b2) * ga * ga
            out.append(a - lr_t * self.m[i] / (np.sqrt(self.v[i]) + dt(self.eps)))
        return out


def actor_ce_step(w, adam, x, a, delta):
    """actor.train_on_batch(s, a_local, sample_weight=delta)
    (agents/resilient_CAC_agents.py:99; Appendix A.5):
    loss = sum_i delta_i * (-log softmax(logits_i)[a_i]) / B, one Keras-Adam step."""
    dt = x.dtype.type
    B = x.shape[0]
    logits, cch = mlp_forward(w, x, cache=True)
    lsm = log_softmax(logits)
    ai = np.asarray(a).reshape(-1).astype(np.int64)
    d = np.asarray(delta, x.dtype).reshape(B)
    ce = -lsm[np.arange(B), ai]
    loss = (d * ce).sum() / dt(B)
    p = np.exp(lsm)
    p[np.arange(B), ai] -= dt(1.0)
    dout = p * (d / dt(B))[:, None]
    g = mlp_backward(w, cch, dout)
    return adam.step(w, g), loss


def actor_fit_minibatch(w, adam, x, a, delta, batch_size, perm):
    """actor.fit(s, a_local, sample_weight=TD, batch_size=200, epochs=1)
    (agents/adversarial_CAC_agents.py:41,116,224)."""
    B = x.shape[0]
    loss_acc, cnt = 0.0, 0
    p = np.asarray(perm)
    d = np.asarray(delta).reshape(B)
    a = np.asarray(a).reshape(B)
    for k in range(0, B, batch_size):
        idx = p[k:k + batch_size]
        w, loss = actor_ce_step(w, adam, x[idx], a[idx], d[idx])
        loss_acc += float(loss) * len(idx)
        cnt += len(idx)
    return w, x.dtype.type(loss_acc / cnt)


# ----------------------------------------------------------------------------
# Resilient aggregation (agents/resilient_CAC_agents.py:42-58; SURVEY 3.4)
# ----------------------------------------------------------------------------
def resilient_aggregation(values_innodes, H):
    v = np.asarray(values_innodes)
    n = v.shape[0]
    own = v[0]
    s = np.sort(v, axis=0)
    lo = np.minimum(s[H], own)
    hi = np.maximum(s[n - H - 1], own)
    clipped = np.maximum(np.minimum(s, hi), lo)          # tf.clip_by_value
    return clipped.mean(axis=0, dtype=v.dtype)


# ----------------------------------------------------------------------------
# Environment (environments/grid_world.py:5-75) -- batched over N envs;
# N == 1 is exactly the reference.
# ----------------------------------------------------------------------------
MOVES = np.array([[0, 0], [-1, 0], [1, 0], [0, -1], [0, 1]], dtype=np.int64)  # grid_world.py:27


class GridWorldOracle:
    def __init__(self, nrow, ncol, n_agents, desired_state, n_envs=1, scaling=True):
        self.nrow, self.ncol, self.n_agents, self.n_envs = nrow, ncol, n_agents, n_envs
        self.desired = np.asarray(desired_state, dtype=np.int64)
        if scaling:                                        # grid_world.py:30-33
            self.mean = np.array([np.mean(np.arange(nrow)), np.mean(np.arange(ncol))])
            self.std = np.array([np.std(np.arange(nrow)), np.std(np.arange(ncol))])
        else:
            self.mean, self.std = np.zeros(2), np.ones(2)
        self.state = np.zeros((n_envs, n_agents, 2), dtype=np.int64)
        self.reward = np.zeros((n_envs, n_agents))

    def set_state(self, state):
        self.state = np.array(state, dtype=np.int64).reshape(self.n_envs, self.n_agents, 2)
        self.reward = np.zeros((self.n_envs, self.n_agents))

    def reset_np_global(self):
        """grid_world.py:37-45 using the NumPy global RNG (N == 1 only)."""
        assert self.n_envs == 1
        self.set_state(np.random.randint([0, 0], [self.nrow, self.ncol],
                                         size=(self.n_agents, 2)))

    def step(self, action):
        """grid_world.py:47-64.  The collision test at :56 includes the agent
        itself, so dist_to_agents == 0 always and the branch at :59-60 is dead;
        agents therefore never interact and the loop vectorises."""
        a = np.asarray(action).astype(np.int64).reshape(self.n_envs, self.n_agents)
        dist = np.abs(self.state - self.desired[None]).sum(-1)           # pre-move
        self.state = np.clip(self.state + MOVES[a], 0, self.nrow - 1)     # :55 (nrow for both coords)
        self.reward = np.where((dist == 0) & (a == 0), 0.0, -dist - 1.0).astype(np.float64)

    def get_data(self):
        """grid_world.py:66-72."""
        return (self.state - self.mean) / self.std, self.reward / 5


# ----------------------------------------------------------------------------
# get_action (agents/resilient_CAC_agents.py:208-219) with injected uniforms
# ----------------------------------------------------------------------------
def sample_action_from_uniforms(probs, u, mu=0.1):
    """Equivalent of the three np.random.choice calls given the three raw
    uniforms they would consume (SURVEY 7 'RNG'):
      choice(n)                 == floor(u0 * n)   (stand-in for randint; exact
                                   parity with MT19937 is not attempted)
      choice(n, p=probs)        == searchsorted(cumsum(p)/sum, u1, 'right')
      choice([a,b], p=[1-mu,mu]) == a if u2 < 1-mu else b
    probs: (..., n_actions); u: (..., 3).  Arithmetic in float32 like the GPU."""
    probs = np.asarray(probs, np.float32)
    n = probs.shape[-1]
    u = np.asarray(u, np.float32)
    rand_a = np.minimum((u[..., 0] * np.float32(n)).astype(np.int64), n - 1)
    cdf = np.cumsum(probs, axis=-1, dtype=np.float32)
    cdf = cdf / cdf[..., -1:]
    pol_a = np.minimum((cdf <= u[..., 1:2]).sum(-1), n - 1)
    return np.where(u[..., 2] < np.float32(1.0 - mu), pol_a, rand_a)


# ----------------------------------------------------------------------------
# Agents
# ----------------------------------------------------------------------------
class RPBCACOracleAgent:
    """agents/resilient_CAC_agents.py:5-223.  Weights are lists of six arrays
    in Keras layout; tensors are (B, n_agents, f) like the reference and are
    flattened internally."""

    def __init__(self, actor_w, critic_w, tr_w, slow_lr, fast_lr, gamma=0.95, H=0,
                 dtype=np.float32):
        self.dtype = dtype
        self.actor = cast_weights(actor_w, dtype)
        self.critic = cast_weights(critic_w, dtype)
        self.TR = cast_weights(tr_w, dtype)
        self.gamma, self.H, self.fast_lr = gamma, H, fast_lr
        self.n_actions = self.actor[4].shape[1]
        self.adam = KerasAdam(slow_lr)

    def _f(self, x):
        return flatten_rows(x, self.dtype)

    def _c(self, y):
        return np.asarray(y, self.dtype).reshape(-1, 1)

    # :60-84
    def critic_update_team(self, s, critic_agg):
        self.critic = self._team(self.critic, self._f(s), self._c(critic_agg))

    def TR_update_team(self, sa, TR_agg):
        self.TR = self._team(self.TR, self._f(sa), self._c(TR_agg))

    def _team(self, w, x, agg):
        dt = self.dtype
        phi = mlp_features(w, x)
        phi_norm = (phi * phi).sum(axis=1) + dt(1.0)
        weights = dt(1.0) / (dt(2.0) * dt(self.fast_lr) * phi_norm)
        new_w, _ = mse_step(w, x, agg, self.fast_lr, sample_weight=weights,
                            last_layer_only=True)
        return new_w

    # :86-101
    def actor_update(self, s, ns, sa, a_local):
        dt = self.dtype
        r_team = mlp_forward(self.TR, self._f(sa))
        V = mlp_forward(self.critic, self._f(s))
        nV = mlp_forward(self.critic, self._f(ns))
        td = r_team + dt(self.gamma) * nV - V
        self.actor, loss = actor_ce_step(self.actor, self.adam, self._f(s), a_local, td)
        return loss

    # :103-140
    def critic_update_local(self, s, ns, r_local):
        dt = self.dtype
        nV = mlp_forward(self.critic, self._f(ns))
        target = self._c(r_local) + dt(self.gamma) * nV
        return fit_fullbatch(self.critic, self._f(s), target, self.fast_lr, 5)

    def TR_update_local(self, sa, r_local):
        return fit_fullbatch(self.TR, self._f(sa), self._c(r_local), self.fast_lr, 5)

    # :142-166
    def resilient_consensus_critic_hidden(self, msgs):
        self.critic = self._hidden(self.critic, msgs)

    def resilient_consensus_TR_hidden(self, msgs):
        self.TR = self._hidden(self.TR, msgs)

    def _hidden(self, w, msgs):
        agg = [resilient_aggregation(np.stack([np.asarray(m[k], self.dtype) for m in msgs]), self.H)
               for k in range(6)]
        return agg[:4] + [w[4], w[5]]                      # weights_agg[:-2] only (:153)

    # :168-206
    def resilient_consensus_critic(self, s, msgs):
        return self._estimates(self.critic, self._f(s), msgs)

    def resilient_consensus_TR(self, sa, msgs):
        return self._estimates(self.TR, self._f(sa), msgs)

    def _estimates(self, w, x, msgs):
        phi = mlp_features(w, x)
        ests = np.stack([phi @ np.asarray(m[4], self.dtype) + np.asarray(m[5], self.dtype)
                         for m in msgs])                   # (n_in, B, 1)
        return resilient_aggregation(ests, self.H)

    # :208-219 -- with injected uniforms
    def action_probs(self, state):
        return softmax(mlp_forward(self.actor, self._f(state)))

    def get_action(self, state, u, mu=0.1):
        return sample_action_from_uniforms(self.action_probs(state), u, mu)

    def get_parameters(self):
        return [self.actor, self.critic, self.TR]


class MaliciousOracleAgent:
    """agents/adversarial_CAC_agents.py:74-182."""

    def __init__(self, actor_w, critic_w, tr_w, slow_lr, fast_lr, gamma=0.95,
                 critic_local_w=None, dtype=np.float32):
        self.dtype = dtype
        self.actor = cast_weights(actor_w, dtype)
        self.critic = cast_weights(critic_w, dtype)
        self.TR = cast_weights(tr_w, dtype)
        self.critic_local_weights = cast_weights(
            critic_w if critic_local_w is None else critic_local_w, dtype)   # :99, main.py:92
        self.gamma, self.fast_lr = gamma, fast_lr
        self.n_actions = self.actor[4].shape[1]
        self.adam = KerasAdam(slow_lr)

    _f = RPBCACOracleAgent._f
    _c = RPBCACOracleAgent._c
    action_probs = RPBCACOracleAgent.action_probs
    get_action = RPBCACOracleAgent.get_action

    def actor_update(self, s, ns, r_local, a_local, perm, batch_size=200):   # :102-119
        dt = self.dtype
        V = mlp_forward(self.critic_local_weights, self._f(s))
        nV = mlp_forward(self.critic_local_weights, self._f(ns))
        td = self._c(r_local) + dt(self.gamma) * nV - V
        self.actor, loss = actor_fit_minibatch(self.actor, self.adam, self._f(s), a_local, td, batch_size, perm)
        return loss

    def critic_update_compromised(self, s, ns, r_comp, perms, batch_size=32):  # :121-135
        dt = self.dtype
        nV = mlp_forward(self.critic, self._f(ns))
        target = self._c(r_comp) + dt(self.gamma) * nV
        self.critic, loss = fit_minibatch(self.critic, self._f(s), target, self.fast_lr, 10, batch_size, perms)
        return self.critic, loss

    def critic_update_local(self, s, ns, r_local, perms, batch_size=32):       # :137-152
        dt = self.dtype
        nV = mlp_forward(self.critic_local_weights, self._f(ns))
        target = self._c(r_local) + dt(self.gamma) * nV
        self.critic_local_weights, _ = fit_minibatch(self.critic_local_weights, self._f(s), target,
                                                     self.fast_lr, 10, batch_size, perms)

    def TR_update_compromised(self, sa, r_comp, perms, batch_size=32):         # :154-165
        self.TR, loss = fit_minibatch(self.TR, self._f(sa), self._c(r_comp), self.fast_lr, 10, batch_size, perms)
        return self.TR, loss

    def get_parameters(self):
        return [self.actor, self.critic, self.TR, self.critic_local_weights]


class GreedyOracleAgent:
    """agents/adversarial_CAC_agents.py:184-275."""

    def __init__(self, actor_w, critic_w, tr_w, slow_lr, fast_lr, gamma=0.95, dtype=np.float32):
        self.dtype = dtype
        self.actor = cast_weights(actor_w, dtype)
        self.critic = cast_weights(critic_w, dtype)
        self.TR = cast_weights(tr_w, dtype)
        self.gamma, self.fast_lr = gamma, fast_lr
        self.n_actions = self.actor[4].shape[1]
        self.adam = KerasAdam(slow_lr)

    _f = RPBCACOracleAgent._f
    _c = RPBCACOracleAgent._c
    action_probs = RPBCACOracleAgent.action_probs
    get_action = RPBCACOracleAgent.get_action

    def actor_update(self, s, ns, r_local, a_local, perm, batch_size=200):   # :211-226
        dt = self.dtype
        V = mlp_forward(self.critic, self._f(s))
        nV = mlp_forward(self.critic, self._f(ns))
        td = self._c(r_local) + dt(self.gamma) * nV - V
        self.actor, loss = actor_fit_minibatch(self.actor, self.adam, self._f(s), a_local, td, batch_size, perm)
        return loss

    def critic_update_local(self, s, ns, r_local, perms, batch_size=32):       # :228-241
        dt = self.dtype
        nV = mlp_forward(self.critic, self._f(ns))
        target = self._c(r_local) + dt(self.gamma) * nV
        self.critic, loss = fit_minibatch(self.critic, self._f(s), target, self.fast_lr, 10, batch_size, perms)
        return self.critic, loss

    def TR_update_local(self, sa, r_local, perms, batch_size=32):              # :243-253
        self.TR, loss = fit_minibatch(self.TR, self._f(sa), self._c(r_local), self.fast_lr, 10, batch_size, perms)
        return self.TR, loss

    def get_parameters(self):
        return [self.actor, self.critic, self.TR]


class FaultyOracleAgent:
    """agents/adversarial_CAC_agents.py:5-72."""

    def __init__(self, actor_w, critic_w, tr_w, slow_lr, gamma=0.95, dtype=np.float32):
        self.dtype = dtype
        self.actor = cast_weights(actor_w, dtype)
        self.critic = cast_weights(critic_w, dtype)
        self.TR = cast_weights(tr_w, dtype)
        self.gamma = gamma
        self.n_actions = self.actor[4].shape[1]
        self.adam = KerasAdam(slow_lr)

    _f = RPBCACOracleAgent._f
    _c = RPBCACOracleAgent._c
    action_probs = RPBCACOracleAgent.action_probs
    get_action = RPBCACOracleAgent.get_action
    actor_update = GreedyOracleAgent.actor_update                        # :28-43 (identical body)

    def get_critic_weights(self):
        return self.critic

    def get_TR_weights(self):
        return self.TR

    def get_parameters(self):
        return [self.actor, self.critic, self.TR]


# ----------------------------------------------------------------------------
# Update round (training/train_agents.py:86-163), batched over N envs.
# Buffer tensors are time-major: row = t * n_envs + e  (SURVEY Appendix C).
# ----------------------------------------------------------------------------
def make_perm_source(seed):
    """Deterministic stand-in for TF's shuffle RNG: returns f(T) -> permutation
    of range(T) (time rows; every env of a time row moves together, Appendix C)."""
    rs = np.random.RandomState(seed)
    return lambda T: rs.permutation(T)


def expand_time_perm(perm_t, n_envs):
    """time-row permutation -> buffer-row permutation (Appendix C)."""
    perm_t = np.asarray(perm_t)
    return (perm_t[:, None] * n_envs + np.arange(n_envs)[None, :]).reshape(-1)


def update_round(agents, labels, in_nodes, s, ns, a, r, *, n_envs, n_epochs, n_actor_steps,
                 common_reward, perm_source):
    """One update round.  s, ns: (B, n_agents, 2); a, r: (B, n_agents, 1).
    n_actor_steps = max_ep_len * n_ep_fixed (time rows used by the actor).
    Returns dict(critic_loss, TR_loss, actor_loss) per agent (np arrays)."""
    n_agents = len(agents)
    dt = agents[0].dtype
    s = np.asarray(s, dt)
    ns = np.asarray(ns, dt)
    a = np.asarray(a, dt)
    r = np.asarray(r, dt)
    B = s.shape[0]
    T = B // n_envs
    sa = np.concatenate([s, a], axis=-1)                                      # :93
    coop = [i for i in range(n_agents) if labels[i] == 'Cooperative']
    n_coop = len(coop)
    r_coop = np.zeros((B, 1), dt)
    for node in coop:                                                          # :96-98
        r_coop = r_coop + r[:, node] / dt(n_coop)
    critic_loss = np.zeros(n_agents)
    TR_loss = np.zeros(n_agents)
    actor_loss = np.zeros(n_agents)

    def perms(n_ep):
        return [expand_time_perm(perm_source(T), n_envs) for _ in range(n_ep)]

    bs = 32 * n_envs                                                           # Appendix C
    for _ in range(n_epochs):                                                  # :100
        critic_msgs, TR_msgs = [], []
        for node in range(n_agents):                                           # :105-121
            r_applied = r_coop if common_reward else r[:, node]
            lab = labels[node]
            if lab == 'Cooperative':
                x, TR_loss[node] = agents[node].TR_update_local(sa, r_applied)
                y, critic_loss[node] = agents[node].critic_update_local(s, ns, r_applied)
            elif lab == 'Greedy':
                x, TR_loss[node] = agents[node].TR_update_local(sa, r[:, node], perms(10), bs)
                y, critic_loss[node] = agents[node].critic_update_local(s, ns, r[:, node], perms(10), bs)
            elif lab == 'Malicious':
                agents[node].critic_update_local(s, ns, r[:, node], perms(10), bs)
                x, TR_loss[node] = agents[node].TR_update_compromised(sa, -r_coop, perms(10), bs)
                y, critic_loss[node] = agents[node].critic_update_compromised(s, ns, -r_coop, perms(10), bs)
            elif lab == 'Faulty':
                x = agents[node].get_TR_weights()
                y = agents[node].get_critic_weights()
            TR_msgs.append(x)
            critic_msgs.append(y)
        for node in coop:                                                      # :125-145
            cm = [critic_msgs[i] for i in in_nodes[node]]
            tm = [TR_msgs[i] for i in in_nodes[node]]
            agents[node].resilient_consensus_critic_hidden(cm)
            agents[node].resilient_consensus_TR_hidden(tm)
            critic_agg = agents[node].resilient_consensus_critic(s, cm)
            TR_agg = agents[node].resilient_consensus_TR(sa, tm)
            agents[node].critic_update_team(s, critic_agg)
            agents[node].TR_update_team(sa, TR_agg)
    na = n_actor_steps * n_envs                                                # :149-153
    Ta = n_actor_steps
    for node in range(n_agents):
        if labels[node] == 'Cooperative':
            actor_loss[node] = agents[node].actor_update(s[-na:], ns[-na:], sa[-na:], a[-na:, node])
        else:
            perm = expand_time_perm(perm_source(min(Ta, T)), n_envs)
            actor_loss[node] = agents[node].actor_update(s[-na:], ns[-na:], r[-na:, node], a[-na:, node], perm,
                                                         200 * n_envs)      # Appendix C: 200 time rows x all envs
    return dict(critic_loss=critic_loss, TR_loss=TR_loss, actor_loss=actor_loss)


def rollout_block(env, agents, labels, *, n_episodes, max_ep_len, gamma, init_states, uniforms, mu=0.1):
    """Episodes under a fixed policy (training/train_agents.py:46-80), batched
    over env.n_envs environments with injected randomness.
      init_states: (n_episodes, n_envs, n_agents, 2) ints  (the reset draws)
      uniforms:    (n_episodes, max_ep_len, n_envs, n_agents, 3) float32
    Returns rows time-major + per-episode logs."""
    N, NA = env.n_envs, env.n_agents
    dt = agents[0].dtype
    S, NS, A, R = [], [], [], []
    est = np.zeros((n_episodes, N, NA))
    ret = np.zeros((n_episodes, N, NA))
    for ep in range(n_episodes):
        env.set_state(init_states[ep])                                         # :55
        state, _ = env.get_data()                                              # :56
        for node in range(NA):                                                 # :60-62
            if labels[node] == 'Cooperative':
                est[ep, :, node] = mlp_forward(agents[node].critic,
                                               flatten_rows(state, dt))[:, 0]
        for j in range(max_ep_len):                                            # :66-80
            action = np.zeros((N, NA))
            for node in range(NA):
                action[:, node] = agents[node].get_action(state, uniforms[ep, j, :, node], mu)
            env.step(action)
            nstate, reward = env.get_data()
            ret[ep] += reward * (gamma ** j)                                   # :71
            S.append(np.array(state))
            NS.append(np.array(nstate))
            A.append(action.reshape(N, NA, 1))
            R.append(np.array(reward).reshape(N, NA, 1))
            state = np.array(nstate)
    cat = lambda L: np.concatenate(L, axis=0)
    return cat(S), cat(NS), cat(A), cat(R), est, ret
