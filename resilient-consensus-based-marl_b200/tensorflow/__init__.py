"""Architecture-descriptor facade for the TensorFlow names the reference driver uses (main.py:7-9,47,60-86).

This is NOT TensorFlow: `keras.Sequential([...])` records the (fixed) RPBCAC network shape and owns a packed
float32 parameter vector in device memory; every forward / backward pass is executed by the sm_90a kernels of
librcmarl.so through rcmarl.ops.  Unsupported Keras functionality raises NotImplementedError."""
import sys
import types

import numpy as np

float32 = np.float32
__version__ = "2.4-rcmarl-facade"


class _Random(types.ModuleType):
    seed = 0

    def set_seed(self, seed):                      # main.py:47
        _Random.seed = int(seed)
        from .keras import _reset_init_rng
        _reset_init_rng(int(seed))


random = _Random("tensorflow.random")
sys.modules["tensorflow.random"] = random


class _Logger:
    def setLevel(self, *_a, **_k):
        pass


def get_logger():                                  # training/train_agents.py:9
    return _Logger()


def convert_to_tensor(value, dtype=None):
    from .keras import Tensor
    from rcmarl import ops
    return Tensor(ops.dev_f32(np.asarray(value, dtype=np.float32) if not hasattr(value, "_t") else value))


def concat(values, axis):
    import torch
    from .keras import Tensor
    from rcmarl import ops
    return Tensor(torch.cat([ops.dev_f32(v) for v in values], dim=axis))


def zeros(shape, dtype=None):
    import torch
    from .keras import Tensor
    return Tensor(torch.zeros(*shape, dtype=torch.float32, device="cuda"))


from . import keras  # noqa: E402,F401
