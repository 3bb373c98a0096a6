"""Host-side logic of the drop-in packages that needs no GPU: the keras-name facade (architecture checks, weight
round trips before any device allocation), agent construction as main.py does it, packing helpers, Keras-Adam step
size, state tables.  (Everything that computes runs in librcmarl.so and is covered by the -m gpu tests.)"""
import numpy as np
import pytest

from golden_util import pretrained


def seq(keras, NA, f, n_out, act, hidden=20, alpha=0.1):
    return keras.Sequential([keras.Input(shape=(NA, f)), keras.layers.Flatten(),
                             keras.layers.Dense(hidden, activation=keras.layers.LeakyReLU(alpha=alpha)),
                             keras.layers.Dense(20, activation=keras.layers.LeakyReLU(alpha=0.1)),
                             keras.layers.Dense(n_out, activation=act)])


def test_facade_models_hold_weights_on_host_until_used():
    import tensorflow as tf
    from tensorflow import keras
    tf.random.set_seed(3)
    m = seq(keras, 5, 2, 1, None)
    assert m.output_shape == (None, 1) and m.n_params == 661 and m._flat is None
    w = m.get_weights()
    assert [a.shape for a in w] == [(10, 20), (20,), (20, 20), (20,), (20, 1), (1,)]
    lim = np.sqrt(6.0 / 30)
    assert np.abs(w[0]).max() <= lim and np.all(w[1] == 0)              # glorot_uniform kernels, zero biases
    tf.random.set_seed(3)
    again = seq(keras, 5, 2, 1, None).get_weights()
    assert all(np.array_equal(a, b) for a, b in zip(w, again))          # tf.random.set_seed makes the init reproducible
    wts, _, _ = pretrained()
    m.set_weights(wts[0][1])
    assert all(np.array_equal(a, b) for a, b in zip(m.get_weights(), wts[0][1])) and m._flat is None
    with pytest.raises(ValueError):
        m.set_weights(wts[0][2])                                        # TR weights do not fit a critic
    # layer-level access used by the reference (res..py:177-184) and the features view (:39-40)
    head = m.layers[-1].get_weights()
    assert head[0].shape == (20, 1) and np.array_equal(head[0], wts[0][1][4])
    m.layers[-1].set_weights([head[0] * 2, head[1]])
    assert np.array_equal(m.get_weights()[4], wts[0][1][4] * 2)
    feat = keras.Model(m.inputs, m.layers[-2].output)
    assert len(feat.get_weights()) == 4
    feat.set_weights([a * 0 for a in feat.get_weights()])
    assert np.all(m.get_weights()[0] == 0) and np.array_equal(m.get_weights()[4], wts[0][1][4] * 2)
    with pytest.raises(NotImplementedError):
        feat(np.zeros((1, 5, 2)))
    with pytest.raises(NotImplementedError):
        m.fit(np.zeros((1, 5, 2)), np.zeros((1, 1)))


def test_facade_rejects_architectures_the_kernels_do_not_implement():
    from tensorflow import keras
    with pytest.raises(NotImplementedError):
        seq(keras, 5, 2, 1, None, hidden=32)
    with pytest.raises(NotImplementedError):
        seq(keras, 5, 2, 1, None, alpha=0.2)
    with pytest.raises(NotImplementedError):
        seq(keras, 5, 2, 3, None)
    with pytest.raises(NotImplementedError):
        keras.Sequential([keras.layers.Flatten(), keras.layers.Dense(20)])


def test_agents_construct_like_main_py_without_touching_the_gpu():
    from tensorflow import keras
    from agents.resilient_CAC_agents import RPBCAC_agent
    from agents.adversarial_CAC_agents import Faulty_CAC_agent, Greedy_CAC_agent, Malicious_CAC_agent
    wts, _, _ = pretrained()
    models = lambda: (seq(keras, 5, 2, 5, 'softmax'), seq(keras, 5, 2, 1, None), seq(keras, 5, 3, 1, None))
    ag = RPBCAC_agent(*models(), slow_lr=0.002, fast_lr=0.01, gamma=0.9, H=1)
    assert (ag.n_actions, ag.H, ag.fast_lr, ag.gamma, ag.n_agents) == (5, 1, 0.01, 0.9, 5) and len(ag.get_parameters()) == 3
    mal = Malicious_CAC_agent(*models(), slow_lr=0.002, fast_lr=0.01, gamma=0.9)
    assert all(np.array_equal(a, b) for a, b in zip(mal.critic_local_weights, mal.critic.get_weights()))   # adversarial:99
    mal.critic_local_weights = wts[4][3]                                 # main.py:92
    assert np.array_equal(mal.get_parameters()[3][0], wts[4][3][0]) and len(mal.get_parameters()) == 4
    assert len(Greedy_CAC_agent(*models(), slow_lr=0.002, fast_lr=0.01).get_parameters()) == 3
    assert len(Faulty_CAC_agent(*models(), slow_lr=0.002).get_parameters()) == 3


def test_packing_and_small_helpers():
    from rcmarl import nets, ops, _lib
    wts, _, _ = pretrained()
    for net, (d_in, n_out) in zip(wts[0], ((10, 5), (10, 1), (15, 1))):
        flat = nets.pack(net)
        assert flat.size == _lib.param_count(d_in, n_out)
        back = nets.unpack(flat, d_in, n_out)
        assert all(np.array_equal(a, b) for a, b in zip(net, back))
    assert nets.n_hidden_params(10) == 640 and nets.n_hidden_params(15) == 740        # SURVEY 8a (a10)
    # Keras Adam: lr_t = lr*sqrt(1-b2^t)/(1-b1^t)  (Appendix A.5)
    assert abs(ops.keras_adam_lr_t(0.002, 1) - 0.002 * np.sqrt(1 - 0.999) / (1 - 0.9)) < 1e-10
    tx, ty = ops.state_tables(5, 5)
    assert tx.dtype == np.float32 and np.allclose(tx, (np.arange(5) - 2) / np.sqrt(2)) and np.array_equal(tx, ty)
    tx10, _ = ops.state_tables(10, 10)
    assert np.allclose(tx10, (np.arange(10) - 4.5) / np.sqrt(8.25))
    # reward table: float32 division by 5 equals the float64 division rounded to float32 for every reachable value
    d = np.arange(0, 40)
    assert np.array_equal((-(d + 1)).astype(np.float32) / np.float32(5), (-(d + 1) / 5.0).astype(np.float32))


def _grid_plan(kinds, n_rows, balanced, na=5, loss=0, sms=148):
    import ctypes as C
    from rcmarl import _lib as L
    k = (C.c_int32 * len(kinds))(*kinds)
    out = (C.c_int32 * len(kinds))()
    L.check(L.lib().rcmarl_grad_grid_plan(na, k, len(kinds), loss, n_rows, int(balanced), sms, out), "rcmarl_grad_grid_plan")
    return list(out)


def test_grad_grid_plan_equal_and_balanced_shares():
    """Host arithmetic of the grad launchers (no device): one wave of at most `sms` CTAs, equal shares by default,
    cost-balanced shares on request (DESIGN.md 4h)."""
    from rcmarl import _lib as L
    SA, S = L.IN_SA, L.IN_S
    # C2 full-batch fit: 4 team-reward + 4 critic jobs over the 12.288 M buffer rows
    assert _grid_plan([SA, S] * 4, 12288000, False) == [18] * 8
    assert _grid_plan([SA, S] * 4, 12288000, True) == [19, 18] * 4
    # C2 mini-batch step of the malicious agent: 131 072 rows, three chains
    assert _grid_plan([S, SA, S], 131072, False) == [49, 49, 49]
    assert _grid_plan([S, SA, S], 131072, True) == [48, 52, 48]          # the team-reward chain drops to 5 rounds
    # tiny inputs: never more CTAs than 8-chunk work units, never fewer than one
    assert _grid_plan([SA, S, S], 100, False) == [1, 1, 1]
    assert _grid_plan([SA, S, S], 100, True) == [1, 1, 1]
    assert _grid_plan([S], 0, False) == [1]
    # one wave whatever the mix
    rs = np.random.RandomState(0)
    for _ in range(200):
        n = int(rs.randint(1, 33))
        kinds = [int(v) for v in rs.randint(0, 3, n)]
        rows = int(rs.randint(0, 1 << 24))
        for na in (5, 16):
            for bal in (False, True):
                g = _grid_plan(kinds, rows, bal, na=na)
                assert min(g) >= 1 and sum(g) <= max(148, n), (kinds, rows, na, bal, g)
    with pytest.raises(L.RcmarlError):
        _grid_plan([7], 10, False)


def test_grad_grid_plan_on_132_sms():
    """The plans the launchers build on an H100 SXM (132 SMs) for the C2 jobs: the full-batch fit and a mini-batch step of the
    malicious agent, equal and cost-balanced shares."""
    from rcmarl import _lib as L
    SA, S = L.IN_SA, L.IN_S
    assert _grid_plan([SA, S] * 4, 12288000, False, sms=132) == [16] * 8
    assert _grid_plan([SA, S] * 4, 12288000, True, sms=132) == [17, 16] * 4
    assert _grid_plan([S, SA, S], 131072, False, sms=132) == [44, 44, 44]
    assert _grid_plan([S, SA, S], 131072, True, sms=132) == [43, 46, 43]
