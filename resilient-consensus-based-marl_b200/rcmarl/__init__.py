"""rcmarl -- host side of the H100-native RPBCAC hot path (see DESIGN.md).

`rcmarl._lib` binds librcmarl.so (C ABI, include/rcmarl.h); `rcmarl.ops` wraps
its entry points for torch CUDA tensors; `rcmarl.trainer` is the batched
training engine used by `training.train_agents.train_RPBCAC`.
"""
__version__ = "0.1"
