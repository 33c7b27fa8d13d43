"""Multi-GPU plumbing: one process per GPU, targets sharded, sources replicated.

The reference has no distributed path at all; this is the multi-GPU design.
``den_n`` is a sum over sources for a fixed target, so with the sources replicated the
first E-step pass needs no communication; the second pass yields per-rank partial sums of the
M-step moments, which are combined by ONE ``ncclAllReduce(sum, float64)`` of 32 doubles per EM
iteration, issued by libcpd_b200.so on its own stream (cpd_comm_init / cpd_em_step).

``torch.distributed`` is used only as the rendezvous: to hand the 128-byte NCCL unique id from
rank 0 to the other ranks.  Any backend works for that (``gloo`` in the CPU tests).
"""
import os

import numpy as np


def shard_bounds(n, rank, world_size):
    """Contiguous, balanced split of n target rows: rank r owns [lo, hi)."""
    return (n * rank) // world_size, (n * (rank + 1)) // world_size


class Communicator(object):
    def __init__(self, rank=0, world_size=1, device=0, exchange=None, gather=None, use_p2p=None):
        """exchange(obj_or_None) -> obj : broadcast of a small picklable object from rank 0.
        gather(obj) -> [obj of rank 0, ..., obj of rank W-1] on every rank (all-gather; also a barrier)."""
        self.rank = int(rank)
        self.world_size = int(world_size)
        self.device = int(device)
        self._exchange = exchange
        self._gather = gather
        self._nccl = None
        # fused NVLink peer-memory exchange of the moments inside the M-step kernel (default) vs ncclAllReduce
        self.use_p2p = (os.environ.get("CPD_B200_NO_P2P", "0") != "1") if use_p2p is None else bool(use_p2p)

    @classmethod
    def from_torch(cls, device=None):
        """Build from an initialised ``torch.distributed`` process group (torchrun env)."""
        import torch.distributed as dist

        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        rank, world = dist.get_rank(), dist.get_world_size()
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", rank))

        def exchange(obj):
            box = [obj]
            dist.broadcast_object_list(box, src=0)
            return box[0]

        def gather(obj):
            box = [None] * world
            dist.all_gather_object(box, obj)
            return box

        return cls(rank, world, device, exchange, gather)

    def shard_bounds(self, n):
        return shard_bounds(n, self.rank, self.world_size)

    def frame_origin(self, target):
        """Common origin every rank centres its shard on: the mean of an evenly strided subsample (at most ~2k points) of the full
        target.  Each rank holds the full host array in this API, so the value is computed locally and is bit-identical
        everywhere; it only has to lie inside the cloud (it is the origin of the FP32 working frame, the moments are exact for
        any origin), and ``ndarray.mean(axis=0)`` over all of a 100k x 3 array costs more host time than an 8-GPU EM iteration."""
        pts = np.asarray(target, dtype=np.float64)
        return pts[:: max(1, pts.shape[0] // 1024)].mean(axis=0)

    def nccl_comm(self):
        """The process's NCCL communicator inside libcpd_b200.so, created on first use (a collective:
        every rank must reach its first use together) and shared by all handles of this process.
        It is deliberately never tied to the lifetime of a Python object: NCCL teardown has
        collective semantics and garbage collection is not synchronised across ranks."""
        if self._nccl is None and self.world_size > 1:
            from . import _cabi

            self._nccl = _cabi.comm_create(self.device, self.world_size, self.rank, self.unique_id())
        return self._nccl

    def attach(self, handle):
        """Wire a _cabi.Handle for multi-rank use (collective: every rank, same order)."""
        if self.world_size <= 1:
            return
        handle.attach_comm(self.nccl_comm(), self.world_size, self.rank)
        if self.use_p2p:
            if self._gather is None:
                raise RuntimeError("Communicator needs a gather function for the P2P exchange")
            from . import _cabi

            handles = self._gather(handle.p2p_local_handle())
            try:
                handle.p2p_attach(handles, self.world_size, self.rank)
                ok, why = True, ""
            except _cabi.CpdError as e:      # e.g. ranks isolated by CUDA_VISIBLE_DEVICES cannot map each other's memory
                ok, why = False, str(e)
            votes = self._gather((ok, why))   # also the barrier: nobody steps before everybody has mapped everybody
            if not all(v[0] for v in votes):
                if ok:
                    handle.p2p_detach()
                self.use_p2p = False          # every rank takes the ncclAllReduce path from here on
                if self.rank == 0:
                    import warnings

                    warnings.warn("probreg_b200: NVLink peer mapping unavailable (%s); using ncclAllReduce for the moments"
                                  % next(v[1] for v in votes if not v[0]))

    def close(self):
        """Collective, optional: destroy the NCCL communicator (all handles must be gone)."""
        if self._nccl is not None:
            from . import _cabi

            _cabi.comm_destroy(self._nccl)
            self._nccl = None

    def unique_id(self):
        """A fresh ncclUniqueId, created on rank 0 and broadcast.  Collective: every rank must
        call it the same number of times, in the same order."""
        from . import _cabi

        uid = _cabi.unique_id() if self.rank == 0 else None
        if self.world_size > 1:
            if self._exchange is None:
                raise RuntimeError("Communicator needs an exchange function when world_size > 1")
            uid = self._exchange(uid)
        return uid
