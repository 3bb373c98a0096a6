"""Keras names used by main.py:60-86 and by the agent constructors, as descriptors over device-resident packed
parameters (see tensorflow/__init__.py).  Network family is fixed by the kernels:
Input(n_agents, f) -> Flatten -> Dense(20, LeakyReLU(0.1)) -> Dense(20, LeakyReLU(0.1)) -> Dense(n_out[, softmax])."""
import sys
import types

import numpy as np

from rcmarl import nets
from rcmarl._lib import HIDDEN, N_ACTIONS, param_count

_init_rng = np.random.RandomState(0)


def _reset_init_rng(seed):
    global _init_rng
    _init_rng = np.random.RandomState(seed)


class Tensor:
    """Device tensor handle with the few operations the reference's call sites use
    (`critic(x)[0][0].numpy()`, training/train_agents.py:62)."""

    def __init__(self, t):
        self._t = t

    def numpy(self):
        a = self._t.detach().cpu().numpy()
        return a[()] if a.ndim == 0 else a

    @property
    def shape(self):
        return tuple(self._t.shape)

    def __getitem__(self, idx):
        return Tensor(self._t[idx])

    def __len__(self):
        return self._t.shape[0]

    def __array__(self, dtype=None, copy=None):
        a = self._t.detach().cpu().numpy()
        return a.astype(dtype) if dtype is not None else a

    def __neg__(self):
        return Tensor(-self._t)


class InputSpec:
    def __init__(self, shape):
        self.shape = tuple(int(x) for x in shape)


def Input(shape=None, **_k):
    return InputSpec(shape)


class LeakyReLU:
    def __init__(self, alpha=0.3):
        self.alpha = float(alpha)


class Flatten:
    def get_weights(self):
        return []

    def set_weights(self, w):
        assert len(w) == 0


class _Sym:
    def __init__(self, model, idx):
        self.model, self.idx = model, idx


class Dense:
    def __init__(self, units, activation=None):
        self.units, self.activation = int(units), activation
        self._model = self._k = None                # bound by Sequential: arrays 2k, 2k+1 of the packed vector

    def get_weights(self):
        return self._model.get_weights()[2 * self._k:2 * self._k + 2]

    def set_weights(self, w):
        allw = self._model.get_weights()
        allw[2 * self._k], allw[2 * self._k + 1] = np.asarray(w[0], np.float32), np.asarray(w[1], np.float32)
        self._model.set_weights(allw)

    @property
    def output(self):
        return _Sym(self._model, self._k)


layers = types.ModuleType("tensorflow.keras.layers")
layers.Flatten, layers.Dense, layers.LeakyReLU, layers.Input = Flatten, Dense, LeakyReLU, Input
sys.modules["tensorflow.keras.layers"] = layers


class _Opt:
    def __init__(self, learning_rate=0.01, **_k):
        self.learning_rate = float(learning_rate)


optimizers = types.ModuleType("tensorflow.keras.optimizers")
optimizers.SGD = type("SGD", (_Opt,), {})
optimizers.Adam = type("Adam", (_Opt,), {})
sys.modules["tensorflow.keras.optimizers"] = optimizers
losses = types.ModuleType("tensorflow.keras.losses")
losses.MeanSquaredError = type("MeanSquaredError", (), {})
losses.SparseCategoricalCrossentropy = type("SparseCategoricalCrossentropy", (), {})
sys.modules["tensorflow.keras.losses"] = losses


class Model:
    """keras.Model(inputs, outputs): a view of a Sequential up to one of its Dense layers (critic_features,
    agents/resilient_CAC_agents.py:39-40).  Shares the parent's parameters."""

    def __init__(self, inputs=None, outputs=None):
        if not isinstance(outputs, _Sym):
            raise NotImplementedError("only Model(model.inputs, model.layers[k].output) is supported")
        self._parent, self._upto = outputs.model, outputs.idx
        self.trainable = True

    def get_weights(self):
        return self._parent.get_weights()[:2 * (self._upto + 1)]

    def set_weights(self, w):
        allw = self._parent.get_weights()
        assert len(w) == 2 * (self._upto + 1)
        allw[:len(w)] = [np.asarray(a, np.float32) for a in w]
        self._parent.set_weights(allw)

    def __call__(self, x):
        raise NotImplementedError("hidden features are computed inside the fused rcmarl_team kernel; "
                                  "they are not materialised (include/rcmarl.h)")


class Sequential(Model):
    def __init__(self, layer_list):
        spec = layer_list[0]
        if not isinstance(spec, InputSpec) or len(spec.shape) != 2:
            raise NotImplementedError("expected keras.Input(shape=(n_agents, n_features)) first (main.py:61)")
        dense = [l for l in layer_list[1:] if isinstance(l, Dense)]
        ok = (len(dense) == 3 and dense[0].units == HIDDEN and dense[1].units == HIDDEN and
              all(isinstance(d.activation, LeakyReLU) and abs(d.activation.alpha - 0.1) < 1e-12 for d in dense[:2]) and
              dense[2].activation in (None, 'softmax') and isinstance(layer_list[1], Flatten))
        if not ok:
            raise NotImplementedError("the sm_90a kernels implement the reference architecture only: "
                                      "Flatten, Dense(20, LeakyReLU(0.1)) x2, Dense(n_out[, softmax]) (main.py:60-82)")
        self.n_agents, self.n_feat = spec.shape
        self.d_in = self.n_agents * self.n_feat
        # the kernels are instantiated for 5 and 16 agents; other team sizes run zero-padded (rcmarl/nets.py)
        self.n_kernel = nets.kernel_agents(self.n_agents)
        self.d_in_k = self.n_kernel * self.n_feat
        self.n_out = dense[2].units
        self.softmax = dense[2].activation == 'softmax'
        if self.n_out not in (1, N_ACTIONS) or self.n_feat not in (2, 3):
            raise NotImplementedError(f"unsupported network shape d_in={self.d_in} n_out={self.n_out}")
        self.layers = list(layer_list[1:])
        for k, d in enumerate(dense):
            d._model, d._k = self, k
        self._host = nets.glorot_uniform(self.d_in, self.n_out, _init_rng)   # Keras default init
        self._flat = None
        self.trainable = True

    # -- parameters ---------------------------------------------------------
    @property
    def n_params(self):
        """Length of the packed DEVICE vector (the kernel instantiation's input width)."""
        return param_count(self.d_in_k, self.n_out)

    @property
    def flat(self):
        """Packed parameters in device memory (allocated on first use)."""
        if self._flat is None:
            import torch
            self._flat = torch.as_tensor(nets.pack_padded(self._host, self.d_in_k)).to("cuda")
            self._host = None
        return self._flat

    def get_weights(self):
        if self._flat is None:
            return [a.copy() for a in self._host]
        return nets.unpack_padded(self._flat.detach().cpu().numpy(), self.d_in, self.d_in_k, self.n_out)

    def set_weights(self, w):
        w = [np.asarray(a, np.float32) for a in w]
        for a, shp in zip(w, nets.shapes(self.d_in, self.n_out)):
            if tuple(a.shape) != tuple(shp):
                raise ValueError(f"weight shape {a.shape} != {shp}")
        if self._flat is None:
            self._host = [a.copy() for a in w]
        else:
            import torch
            self._flat.copy_(torch.as_tensor(nets.pack_padded(w, self.d_in_k)))

    @property
    def inputs(self):
        return [_Sym(self, -1)]

    @property
    def output_shape(self):
        return (None, self.n_out)

    # -- execution ----------------------------------------------------------
    def _forward(self, x):
        import torch
        from rcmarl import ops, _lib as L
        x = ops.dev_f32(x)
        B = x.shape[0]
        x = x.reshape(B, -1)
        if x.shape[1] != self.d_in:
            raise ValueError(f"expected input with {self.d_in} features per row, got {x.shape[1]}")
        out = torch.empty(B, self.n_out, dtype=torch.float32, device=x.device)
        x = nets.pad_agent_slots(x, self.n_agents, self.n_kernel)
        if self.n_feat == 3:
            rows, kind = ops.make_rows(x, None, None, self.n_kernel), L.IN_SA
        else:
            rows, kind = ops.make_rows(None, x, None, self.n_kernel), L.IN_NS
        ops.values(rows, [ops.value_job(out, [(self.flat, kind, 1.0)], n_out=self.n_out, softmax=int(self.softmax))])
        return out

    def __call__(self, x):
        return Tensor(self._forward(x))

    def predict(self, x, **_k):
        return self._forward(x).cpu().numpy()

    def compile(self, optimizer=None, loss=None, **_k):
        self.optimizer, self.loss = optimizer, loss

    def fit(self, *a, **k):
        raise NotImplementedError("use the agent methods (critic_update_local, ...) or rcmarl.trainer: training runs "
                                  "in the fused sm_90a kernels, not through a generic Keras fit loop")

    train_on_batch = fit


sys.modules["tensorflow.keras"] = sys.modules[__name__]
