"""Data-parallel plumbing of the TD update (SURVEY.md 8e): parameters, optimizer state and
target networks are replicated on every rank, the global minibatch is split into equal
contiguous row shards, and ONE all-reduce of the flat gradient arena per optimizer sub-step
turns per-shard mean-loss gradients into the global-batch gradient (every loss of the path is
a batch mean: dqn_trainer_base.py:146-155, qrdqn_trainer.py:153-155, sac_trainer.py:242,280,
td3_trainer.py:157,184).  Adam and the Polyak update then run redundantly and identically
on all ranks -- no broadcast.  The reference itself has no collective on this path
(docs/distributed.rst:12-22 only documents the intent)."""
from typing import Tuple

import torch


def shard_rows(batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous row range [lo, hi) of `rank`; requires world | batch so that the mean of
    shard means equals the global mean."""
    if batch % world != 0:
        raise ValueError(f"global batch {batch} is not divisible by world size {world}")
    per = batch // world
    return rank * per, (rank + 1) * per


def allreduce_mean_(flat_grad: torch.Tensor, group=None) -> float:
    """In-place SUM all-reduce of the flat gradient; returns the 1/world scale the fused Adam
    applies while it reads the gradient (no extra pass over it)."""
    import torch.distributed as dist

    dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return 1.0 / dist.get_world_size(group)


# ---------------------------------------------------------------------------
# Gradient exchange fused into the optimizer kernel over NVLink peer memory
# ---------------------------------------------------------------------------
class P2PExchange:
    """Peer-mapped receive buffers for `rb200_adam_soft_update`'s fused data-parallel step
    (include/reagent_b200.h, rb200_adam_args_t.dp_*): one IPC-exported pool per rank, mapped
    into every peer process of `group` (one process per GPU of one NVLink/NVSwitch node),
    carved identically on all ranks -- one slice per optimizer.  With it a DP update needs no
    NCCL call and no separate gradient-reduce launch: the Adam kernel of every rank pushes its
    gradient slice to the peers, waits for theirs and sums them in rank order."""

    MAX_BLOCKS = 132 * 4  # rb200_adam_blocks(): four blocks per SM of an H100

    def __init__(self, group=None, pool_bytes: int = 512 << 20):
        import ctypes as C

        import torch.distributed as dist

        from .. import _lib

        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.pool_bytes = int(pool_bytes)
        lib = _lib.lib()
        base = C.c_void_p()
        _lib.check(lib.rb200_dp_alloc(self.pool_bytes, C.byref(base)), "rb200_dp_alloc")
        self.base = int(base.value)
        h = (C.c_ubyte * 64)()
        _lib.check(lib.rb200_dp_ipc_handle(self.base, h), "rb200_dp_ipc_handle")
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(h), group=group)
        self.peer_base = []
        for r, hb in enumerate(handles):
            if r == self.rank:
                self.peer_base.append(self.base)
                continue
            buf = (C.c_ubyte * 64).from_buffer_copy(hb)
            p = C.c_void_p()
            _lib.check(lib.rb200_dp_ipc_open(buf, C.byref(p)), f"rb200_dp_ipc_open(rank {r})")
            self.peer_base.append(int(p.value))
        self._off = 0
        self._slices = {}
        dist.barrier(group=group)  # every pool is allocated, zeroed and mapped before any push

    def _carve(self, recv_bytes: int, flag_bytes: int):
        """(recv pointer table, flag pointer table) of the next free range of every rank's pool;
        identical on all ranks as long as they carve in the same order."""
        off = (self._off + 255) // 256 * 256
        if off + recv_bytes + flag_bytes > self.pool_bytes:
            raise RuntimeError("P2PExchange pool exhausted: raise pool_bytes")
        self._off = off + recv_bytes + flag_bytes
        dev = torch.device("cuda", torch.cuda.current_device())
        recv = torch.tensor([b + off for b in self.peer_base], dtype=torch.int64, device=dev)
        flags = torch.tensor([b + off + recv_bytes for b in self.peer_base], dtype=torch.int64,
                             device=dev)
        return recv, flags

    def slice_for(self, key, n: int):
        """(recv pointer table, flag pointer table, stride, max_blocks) for the optimizer `key`
        (call in the same order on every rank)."""
        if key in self._slices:
            return self._slices[key]
        W = self.world
        stride = (int(n) + 31) // 32 * 32
        recv, flags = self._carve(2 * W * stride * 4, 2 * W * self.MAX_BLOCKS * 4)
        s = (recv, flags, stride, self.MAX_BLOCKS)
        self._slices[key] = s
        return s

    def priority_slice(self, key, batch_global: int):
        """(recv pointer table, flag pointer table, epoch counter) of `rb200_per_priority_exchange`
        for the prioritized update `key` of `batch_global` rows: a fp64 [2][batch_global]
        receive buffer and uint32 [2][world] flags per rank, next to the optimizer slices (call
        in the same order on every rank).  The epoch is this rank's own device counter."""
        if key in self._slices:
            return self._slices[key]
        recv, flags = self._carve(2 * int(batch_global) * 8, 2 * self.world * 4)
        epoch = torch.zeros(1, dtype=torch.int32, device=recv.device)
        s = (recv, flags, epoch)
        self._slices[key] = s
        return s


_EXCHANGES = {}


def enable_p2p(group=None, pool_bytes: int = 512 << 20) -> P2PExchange:
    """Create (once per process group) the peer-memory exchange; afterwards `dp_fused_step`
    uses the fused kernel instead of reduce + NCCL all-reduce + Adam."""
    key = id(group) if group is not None else 0
    if key not in _EXCHANGES:
        _EXCHANGES[key] = P2PExchange(group, pool_bytes)
    return _EXCHANGES[key]


def p2p_for(group):
    return _EXCHANGES.get(id(group) if group is not None else 0)


def dp_fused_step(opt, process_group, **kw):
    """One optimizer sub-step of a data-parallel update.  `process_group` None: single rank.
    With a P2P exchange enabled for the group: ONE launch (gradient exchange fused into the
    Adam kernel over NVLink peer memory).  Otherwise: rb200_grad_reduce + NCCL all-reduce +
    Adam (the plain collective path)."""
    if process_group is None:
        return opt.fused_step(**kw)
    ex = p2p_for(process_group)
    if ex is not None:
        return opt.fused_step(dp=ex, **kw)
    from .workspace import reduced_grad

    g = reduced_grad(opt.arena)
    scale = allreduce_mean_(g, process_group)
    return opt.fused_step(grad=g, grad_scale=scale, **kw)
