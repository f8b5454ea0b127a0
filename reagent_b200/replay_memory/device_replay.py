"""Device-resident mode of the (Prioritized)ReplayBuffer (SURVEY.md 8f rank 1).

`DeviceReplay(rb)` takes over the bookkeeping of an existing buffer: validity, cursor / episode
counters, the fp64 sum tree and -- for index selection -- a copy of CPython's MT19937 state
live ON THE GPU from then on, and three single-CTA kernels restate the reference's host logic
with identical results (csrc/rb200_replay_dev.cu):

    add()            ReplayBuffer.add, stack_size == 1        circular_replay_buffer.py:468-547
    set_priority()   SumTree.set in order                     sum_tree.py:164-189
    draw_indices()   PrioritizedReplayBuffer.sample_index_batch (stratified random.uniform draws,
                     tree descents, sequential retries)        prioritized_replay_buffer.py:86-115

so that an online loop "add a transition -> draw a minibatch -> train" needs no host work per
step beyond writing the new transition into pinned memory (training/fused_step.py captures
the whole step in one CUDA graph).  `sync_to_host()` brings the host mirrors (and Python's
`random` state) back, after which the buffer's ordinary host-side API continues the same
streams bit for bit.
"""
import itertools
import math
import random
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch

from .. import _lib

MAX_ADD = 1024  # transitions per rb200_replay_add_device launch
_EXCHANGE_KEYS = itertools.count()  # peer-memory priority slices, in the order of first use


@dataclass(frozen=True)
class PrioritizedUpdate:
    """Prioritized experience replay (Schaul et al. 2016) for FusedDqnStep: after each update the
    drawn transitions get p_i = (|TD error_i| + eps) ** alpha, and the update is weighted by
    w_i = (p_min / p_i) ** beta_t (p over the drawn leaves, p_min their smallest nonzero one),
    beta_t = min(1, beta0 + (1 - beta0) * t / beta_updates) with t the optimizer's step count."""
    alpha: float = 0.6
    beta0: float = 0.4
    beta_updates: int = 100_000
    eps: float = 1e-6

    def __post_init__(self):
        if not (math.isfinite(self.alpha) and self.alpha >= 0.0):
            raise ValueError(f"alpha must be finite and >= 0, got {self.alpha}")
        if not (math.isfinite(self.eps) and self.eps >= 0.0):
            raise ValueError(f"eps must be finite and >= 0, got {self.eps}")
        if not 0.0 <= self.beta0 <= 1.0:
            raise ValueError(f"beta0 must lie in [0, 1], got {self.beta0}")
        if not (math.isfinite(self.beta_updates) and self.beta_updates > 0):
            raise ValueError(f"beta_updates must be positive, got {self.beta_updates}")


@dataclass(frozen=True)
class PriorityShard:
    """This rank's place in a data-parallel prioritized update: its rows are
    [row0, row0 + n) of the `batch_global` drawn ones, and `group` is the process group whose
    ranks hold the others (None: one rank).  The priorities of all rows are gathered on every
    rank -- over NVLink peer memory when `enable_p2p(group)` ran, else by NCCL all-gather -- and
    every rank applies the same vector to its replicated tree."""
    row0: int
    batch_global: int
    group: object = None


class DeviceReplay:
    def __init__(self, rb, stage_rows: int = 1, stage_slots: int = 1):
        if rb._stack_size != 1:
            raise NotImplementedError("device-resident replay needs stack_size == 1")
        if not rb._initialized_buffer:
            raise RuntimeError("add at least one transition (or add_batch) before going device-resident")
        rb._flush()
        self.rb = rb
        self.dev = dev = rb._dev()
        self.prioritized = hasattr(rb, "sum_tree")
        self.state = torch.tensor([int(rb.add_count), int(rb._num_transitions_in_current_episode),
                                   int(rb._num_valid_indices), 0], dtype=torch.int64, device=dev)
        self.status = torch.zeros(2, dtype=torch.int32, device=dev)
        self.tree = self.max_priority = self.mt_state = None
        if self.prioritized:
            self.tree = rb.sum_tree.device_heap(dev)
            self.max_priority = torch.tensor([rb.sum_tree.max_recorded_priority],
                                             dtype=torch.float64, device=dev)
            self.upload_host_rng()
        self._bounds = {}
        self._exchange_key = None
        self._keys = [e.name for e in rb.get_add_args_signature()
                      if e.name not in ("terminal", "reward", "priority")]
        self._alloc_stage(stage_rows, stage_slots)
        rb._device_resident = self

    # ---- staging ---------------------------------------------------------------
    def _alloc_stage(self, rows: int, slots: int = 1):
        """`slots` independent staging blocks of `rows` transitions each.  A block is ONE
        contiguous pinned buffer (key after key, 16-byte aligned), mirrored on the device, so
        that an add is a single host->device copy however many keys a transition has."""
        rb = self.rb
        self.stage_rows, self.stage_slots = rows, slots
        self._layout = {}
        off = 0
        for e in rb.get_add_args_signature():
            md = e.metadata
            if e.name == "priority":
                dt, shape = np.dtype(np.float64), ()
            else:
                dt, shape = np.dtype(md.dtype), tuple(md.shape)
            nbytes = rows * int(np.prod(shape, dtype=np.int64)) * dt.itemsize
            self._layout[e.name] = (off, dt, shape, nbytes)
            off = (off + nbytes + 15) // 16 * 16
        self.block_bytes = off
        self.host_raw = torch.zeros(slots, off, dtype=torch.uint8).pin_memory()
        self.dev_raw = torch.zeros(slots, off, dtype=torch.uint8, device=self.dev)
        raw = self.host_raw.numpy()
        # numpy views of the pinned block: a per-step `stage()` costs ~1 us
        self.host_np = [{k: raw[sl, o:o + nb].view(dt).reshape((rows,) + shape)
                         for k, (o, dt, shape, nb) in self._layout.items()}
                        for sl in range(slots)]

    def rb_desc(self) -> _lib.ReplayDevT:
        rb = self.rb
        d = _lib.ReplayDevT()
        d.state = self.state.data_ptr()
        d.capacity = rb._replay_capacity
        d.update_horizon = rb._update_horizon
        d.valid = rb._valid_dev.data_ptr()
        d.terminal = rb._store["terminal"].data_ptr()
        d.reward = rb._store["reward"].data_ptr()
        if self.prioritized:
            d.tree = self.tree.data_ptr()
            d.tree_depth = rb.sum_tree.depth
            d.max_priority = self.max_priority.data_ptr()
        return d

    def stage(self, row: int, slot: int = 0, priority_from_max: bool = False, **transition):
        """Write one transition into row `row` of staging block `slot` (host only).  With
        `priority_from_max` (prioritized replay) a transition without `priority` is staged as NaN,
        which an add launched with `priority_from_max` replaces by the largest priority recorded
        so far, read on the device when it is inserted."""
        views = self.host_np[slot]
        if priority_from_max and "priority" not in transition:
            views["priority"][row] = np.nan
        for k, v in transition.items():
            views[k][row] = v

    def launch_add(self, n: int, slot: int = 0, priority_from_max: bool = False):
        """ONE host->device copy of staging block `slot` + the add kernel for its first `n`
        rows, on the current stream (graph-capturable: fixed pinned / device addresses).
        `priority_from_max`: a NaN staged priority means the largest one recorded so far."""
        assert 1 <= n <= min(self.stage_rows, MAX_ADD) and 0 <= slot < self.stage_slots
        self.dev_raw[slot].copy_(self.host_raw[slot], non_blocking=True)
        base = self.dev_raw[slot].data_ptr()
        a = _lib.AddArgsT()
        a.rb = self.rb_desc()
        a.n = n
        a.terminal_in = base + self._layout["terminal"][0]
        a.reward_in = base + self._layout["reward"][0]
        a.priority_in = base + self._layout["priority"][0] if self.prioritized else None
        for j, k in enumerate(self._keys):
            md = self.rb._key_to_replay_elem[k].metadata
            a.rows[j].src = base + self._layout[k][0]
            a.rows[j].dst = self.rb._store[k].data_ptr()
            a.rows[j].row_bytes = md.row_bytes
            a.rows[j].which = 0
        a.n_rows = len(self._keys)
        a.priority_from_max = int(bool(priority_from_max))
        _lib.check(_lib.lib().rb200_replay_add_device(a, _lib.cur_stream()), "rb200_replay_add_device")
        self.rb._valid_index_stale = True

    @property
    def h2d_bytes_per_add(self) -> int:
        """Bytes of the single host->device copy of one add launch (one staging block)."""
        return self.block_bytes

    def add(self, **transition):
        """ReplayBuffer.add (one transition) on the device."""
        self.stage(0, 0, **transition)
        self.launch_add(1)

    def add_rows(self, **arrays):
        """n consecutive add() calls from arrays with a leading dimension n."""
        n = len(arrays["terminal"])
        if n > self.stage_rows and self.stage_rows < MAX_ADD:
            self._alloc_stage(min(MAX_ADD, n), self.stage_slots)
        for s0 in range(0, n, self.stage_rows):
            m = min(self.stage_rows, n - s0)
            for k, v in arrays.items():
                self.host_np[0][k][:m] = np.asarray(v)[s0:s0 + m]
            self.launch_add(m)
            torch.cuda.current_stream().synchronize()  # the pinned block is reused

    # ---- priorities ----------------------------------------------------------------
    def set_priority(self, indices, priorities):
        """PrioritizedReplayBuffer.set_priority (prioritized_replay_buffer.py:149-160) on the
        device tree; indices / priorities may be host arrays or device tensors."""
        idx = torch.as_tensor(indices).to(self.dev, torch.int64).contiguous()
        val = torch.as_tensor(priorities).to(self.dev, torch.float64).reshape(-1).contiguous()
        rc = _lib.lib().rb200_sumtree_set_device(
            self.tree.data_ptr(), self.rb.sum_tree.depth, idx.data_ptr(), val.data_ptr(),
            idx.numel(), self.max_priority.data_ptr(), self.status.data_ptr(), _lib.cur_stream())
        _lib.check(rc, "rb200_sumtree_set_device")
        self._keep = (idx, val)

    def importance_weights(self, indices: torch.Tensor, step: torch.Tensor, per: PrioritizedUpdate,
                           out: torch.Tensor, out64: Optional[torch.Tensor] = None):
        """PER importance weights of the drawn `indices` from the current leaves (fp32 `out`,
        optionally fp64 `out64`); `step` is the optimizer's int64 device step counter."""
        rc = _lib.lib().rb200_per_weights(
            self.tree.data_ptr(), self.rb.sum_tree.depth, indices.data_ptr(), indices.numel(),
            step.data_ptr(), float(per.beta0), float(per.beta_updates), out.data_ptr(),
            None if out64 is None else out64.data_ptr(), _lib.cur_stream())
        _lib.check(rc, "rb200_per_weights")
        return out

    def write_back_priorities(self, indices: torch.Tensor, td_target: torch.Tensor,
                              q_selected: torch.Tensor, per: PrioritizedUpdate,
                              p_out: torch.Tensor, shard: Optional[PriorityShard] = None):
        """set_priority(indices, (|q_selected - td_target| + eps) ** alpha), in batch order; the
        priorities also go to `p_out` (fp64).  A non-finite one applies none (status 3).
        With `shard`, td_target / q_selected are this rank's rows of the global update, and
        `indices` and `p_out` have all `shard.batch_global` of them (p_out: the gathered
        priorities, the same on every rank)."""
        if shard is not None:
            a = _lib.PerExchangeArgsT()
            a.td_target, a.q_selected = td_target.data_ptr(), q_selected.data_ptr()
            return self._sharded_write_back(a, indices, td_target.numel(), per, p_out, shard)
        rc = _lib.lib().rb200_per_priority_update(
            self.tree.data_ptr(), self.rb.sum_tree.depth, indices.data_ptr(), td_target.data_ptr(),
            q_selected.data_ptr(), indices.numel(), float(per.alpha), float(per.eps),
            p_out.data_ptr(), self.max_priority.data_ptr(), self.status.data_ptr(),
            _lib.cur_stream())
        _lib.check(rc, "rb200_per_priority_update")
        return p_out

    def write_back_row_priorities(self, indices: torch.Tensor, row_loss: torch.Tensor,
                                  divisor: float, per: PrioritizedUpdate, p_out: torch.Tensor,
                                  shard: Optional[PriorityShard] = None):
        """set_priority(indices, (|row_loss| / divisor + eps) ** alpha), in batch order, for the
        distributional heads, whose priority is the row's own loss (fp32 `row_loss`, fp64
        arithmetic); the priorities also go to `p_out` (fp64).  A non-finite one applies none
        (status 3).  `shard`: as write_back_priorities."""
        if shard is not None:
            a = _lib.PerExchangeArgsT()
            a.row_loss, a.divisor = row_loss.data_ptr(), float(divisor)
            return self._sharded_write_back(a, indices, row_loss.numel(), per, p_out, shard)
        rc = _lib.lib().rb200_per_priority_update_rows(
            self.tree.data_ptr(), self.rb.sum_tree.depth, indices.data_ptr(), row_loss.data_ptr(),
            indices.numel(), float(divisor), float(per.alpha), float(per.eps), p_out.data_ptr(),
            self.max_priority.data_ptr(), self.status.data_ptr(), _lib.cur_stream())
        _lib.check(rc, "rb200_per_priority_update_rows")
        return p_out

    def _sharded_write_back(self, a, indices, n_local: int, per: PrioritizedUpdate,
                            p_out: torch.Tensor, shard: PriorityShard):
        """Gather every rank's priorities into p_out (the exchange args `a` carry this rank's
        sources), then apply them all in global batch order."""
        from ..training.data_parallel import p2p_for

        lib = _lib.lib()
        a.alpha, a.eps = float(per.alpha), float(per.eps)
        a.n_local, a.row0, a.B_global = n_local, shard.row0, shard.batch_global
        a.world, a.rank = 1, 0
        ex = None if shard.group is None else p2p_for(shard.group)
        if shard.group is None or ex is not None:
            if ex is not None:
                if self._exchange_key is None:  # first sharded write-back: same order on all ranks
                    self._exchange_key = ("per", next(_EXCHANGE_KEYS))
                recv, flags, epoch = ex.priority_slice(self._exchange_key, shard.batch_global)
                a.world, a.rank = ex.world, ex.rank
                a.recv, a.flags, a.epoch = recv.data_ptr(), flags.data_ptr(), epoch.data_ptr()
            a.out = p_out.data_ptr()
            _lib.check(lib.rb200_per_priority_exchange(a, _lib.cur_stream()),
                       "rb200_per_priority_exchange")
        else:
            import torch.distributed as dist

            local = self._local_priorities(n_local)
            a.row0, a.B_global, a.out = 0, n_local, local.data_ptr()
            _lib.check(lib.rb200_per_priority_exchange(a, _lib.cur_stream()),
                       "rb200_per_priority_exchange")
            dist.all_gather_into_tensor(p_out, local, group=shard.group)
        rc = lib.rb200_per_priority_apply(
            self.tree.data_ptr(), self.rb.sum_tree.depth, indices.data_ptr(), p_out.data_ptr(),
            indices.numel(), self.max_priority.data_ptr(), self.status.data_ptr(),
            _lib.cur_stream())
        _lib.check(rc, "rb200_per_priority_apply")
        return p_out

    def _local_priorities(self, n: int) -> torch.Tensor:
        """This rank's fp64 priorities before an NCCL all-gather (one fixed buffer: graph-safe)."""
        buf = getattr(self, "_local_prio", None)
        if buf is None or buf.numel() != n:
            buf = self._local_prio = torch.empty(n, dtype=torch.float64, device=self.dev)
        return buf

    # ---- index selection ---------------------------------------------------------------
    def upload_host_rng(self):
        """Python's `random` state -> device (the device stream continues it).  The 624 words +
        position travel as the int32 bit patterns of CPython's uint32 values."""
        _, internal, _ = random.getstate()
        words = np.asarray(internal, dtype=np.uint32)
        self.mt_state = torch.from_numpy(words.view(np.int32).copy()).to(self.dev)

    def _bounds_for(self, B: int):
        b = self._bounds.get(B)
        if b is None:
            lin = np.linspace(0.0, 1.0, B + 1)  # sum_tree.py:149
            b = (torch.from_numpy(np.ascontiguousarray(lin[:-1])).to(self.dev),
                 torch.from_numpy(np.ascontiguousarray(lin[1:])).to(self.dev))
            self._bounds[B] = b
        return b

    def draw_indices(self, batch_size: int, out: Optional[torch.Tensor] = None,
                     queries_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """sample_index_batch(batch_size) of the prioritized buffer, entirely on the device."""
        if not self.prioritized:
            raise NotImplementedError("device index selection covers the prioritized buffer")
        lo, hi = self._bounds_for(batch_size)
        if out is None:
            out = torch.empty(batch_size, dtype=torch.int64, device=self.dev)
        a = _lib.PerDrawArgsT()
        a.mt_state = self.mt_state.data_ptr()
        a.batch = batch_size
        a.lo, a.hi = lo.data_ptr(), hi.data_ptr()
        a.tree = self.tree.data_ptr()
        a.tree_depth = self.rb.sum_tree.depth
        a.valid = self.rb._valid_dev.data_ptr()
        a.max_attempts = int(self.rb._max_sample_attempts)
        a.indices_out = out.data_ptr()
        a.queries_out = None if queries_out is None else queries_out.data_ptr()
        a.status = self.status.data_ptr()
        _lib.check(_lib.lib().rb200_per_draw_indices(a, _lib.cur_stream()), "rb200_per_draw_indices")
        return out

    # ---- errors / host mirrors ---------------------------------------------------------------
    def raise_if_failed(self, status_host=None):
        """Turn the sticky device status into the reference's exceptions (synchronises unless a
        host copy of the status words is given)."""
        if status_host is None:
            st = self.status.cpu()
            code = max(int(st[0]), int(self.state[3].item()))
        else:
            code = int(status_host[0])
        if code == 1:
            raise RuntimeError(
                "Max sample attempts: Tried {} times but could not sample a valid index "
                "for every stratum.".format(self.rb._max_sample_attempts))
        if code == 2:
            raise ValueError("Sum tree values should be nonnegative.")
        if code == 3:
            raise FloatingPointError(
                "prioritized replay: a TD error or row loss was not finite, so its priority "
                "could not be "
                "written back (no priority of that update was applied)")

    def sync_to_host(self):
        """Bring the host-side mirrors (counters, validity, terminal flags, sum tree, Python's
        `random` state) up to date and hand the bookkeeping back to the host API."""
        rb = self.rb
        torch.cuda.synchronize(self.dev)
        st = self.state.cpu().tolist()
        rb.add_count = np.array(int(st[0]))
        rb._num_transitions_in_current_episode = int(st[1])
        rb._num_valid_indices = int(st[2])
        rb._is_index_valid.copy_(rb._valid_dev.cpu().bool())
        rb._terminal_host[:] = rb._store["terminal"].cpu().numpy().astype(np.bool_)
        rb._valid_dirty = []
        rb._valid_index_stale = True
        if self.prioritized:
            t = rb.sum_tree
            t.heap[:] = self.tree.cpu().numpy()
            t.max_recorded_priority = float(self.max_priority.item())
            t._dirty = []
            t.version = getattr(t, "version", 0) + 1
            rb._post_add_batch()  # recompute the invalid-but-positive set
            words = self.mt_state.cpu().numpy().view(np.uint32)
            ver, _, gauss = random.getstate()
            random.setstate((ver, tuple(int(w) for w in words), gauss))
        rb._device_resident = None
