"""Peer-memory exchange context for data-parallel training on one node (include/rcmarl.h, csrc/comm.cuh):
each rank allocates an exchange buffer, the CUDA IPC handles are swapped through torch.distributed (plumbing), and the
context is bound so that rcmarl_grad / rcmarl_team / rcmarl_minibatch_fit reduce across GPUs inside their own kernels
over NVLink -- no NCCL call per optimisation step."""
import ctypes as C

import torch

from . import _lib as L


class PeerComm:
    def __init__(self, rank, world, group=None, max_floats=L.MAX_JOBS * 1536):
        import torch.distributed as dist
        lib = L.lib()
        self.rank, self.world = rank, world
        h = C.c_void_p()
        nb = lib.rcmarl_comm_handle_bytes()
        buf = C.create_string_buffer(nb)
        # create + export may fail on one rank only (out of memory, IPC disabled): every rank still takes part in the
        # gather below and all of them see the failure, so the collectives stay matched and nobody hangs
        st = lib.rcmarl_comm_create(rank, world, max_floats, C.byref(h))
        if st == 0:
            st = lib.rcmarl_comm_export(h, buf)
        self.handle = h if h.value else None
        gathered = [None] * world
        dist.all_gather_object(gathered, (int(st), bytes(buf.raw)), group=group)
        if any(g[0] != 0 for g in gathered):
            if self.handle is not None:
                lib.rcmarl_comm_destroy(self.handle)
                self.handle = None
            bad = [r for r, g in enumerate(gathered) if g[0] != 0]
            raise L.RcmarlError(f"rcmarl_comm_create / export failed on rank(s) {bad}")
        status = lib.rcmarl_comm_connect(h, b"".join(g[1] for g in gathered))
        torch.cuda.synchronize()
        dist.barrier(group=group)                     # every rank has mapped (or failed to map) every buffer
        if status != 0:
            lib.rcmarl_comm_destroy(h)
            self.handle = None
            L.check(status, "rcmarl_comm_connect")
        L.check(lib.rcmarl_comm_bind(h), "rcmarl_comm_bind")
        self.bound = True

    def check(self):
        """Raise if a peer wait timed out inside a kernel (synchronises the device)."""
        if L.lib().rcmarl_comm_error(self.handle) != 0:
            raise L.RcmarlError("peer-memory all-reduce timed out waiting for another rank")

    def close(self):
        if self.handle is not None:
            lib = L.lib()
            torch.cuda.synchronize()
            lib.rcmarl_comm_bind(None)
            lib.rcmarl_comm_destroy(self.handle)
            self.handle, self.bound = None, False
