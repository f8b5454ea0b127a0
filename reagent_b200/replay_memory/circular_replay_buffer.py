"""ReplayBuffer with the reference's API (reagent/replay_memory/circular_replay_buffer.py:
307-890) over DEVICE-resident storage.

Host side (this file) keeps exactly the reference's bookkeeping -- cursor, episode length,
validity (`_is_index_valid`), zero-padding at episode starts, the terminal look-back
(:468-522) -- and stages added transitions in pinned memory; `_flush()` moves them into
`_store[key]` (CUDA tensors, [capacity, *shape]) with at most two contiguous copies per key.
Sampling is ONE fused CUDA launch (rb200_replay_sample): index selection, n-step reward
fold, segment gather, optional dense-feature normalisation and trainer-batch formatting.

Out of scope (raise NotImplementedError): sparse id-list elements (IDListMetadata /
IDScoreListMetadata, :143-282) and `return_as_timeline_format` (python lists of ragged
tensors, :719-730).
"""
import collections
import gzip
import logging
import os
import pickle
from typing import Dict, List, Optional

import numpy as np
import torch

from .. import _lib

logger = logging.getLogger(__name__)

STORE_FILENAME_PREFIX = "$store$_"
CHECKPOINT_DURATION = 4
REQUIRED_KEYS = ["observation", "action", "reward", "terminal"]
_STAGE_ROWS = 4096


class DenseMetadata:
    """shape/dtype of one replay element (circular_replay_buffer.py:88-141)."""

    def __init__(self, name, example):
        if isinstance(example, (dict, torch.Tensor)):
            if isinstance(example, dict):
                raise NotImplementedError(
                    f"{name}: sparse id-list replay elements are out of scope of reagent_b200")
            raise AssertionError(f"{name}: {type(example)} is dict or torch.Tensor")
        arr = np.array(example)
        dtype = arr.dtype
        if dtype == np.dtype("float64"):
            dtype = np.dtype("float32")
        if dtype == object:
            raise ValueError(f"Unable to deduce type for {name}: {example}")
        self.name = name
        self.shape = arr.shape
        self.dtype = dtype

    def validate(self, name, input):
        assert not isinstance(input, (dict, torch.Tensor)), (
            f"{name}: {type(input)} is dict or torch.Tensor")
        arr = np.array(input)
        dtype = arr.dtype
        if dtype == np.dtype("float64"):
            dtype = np.dtype("float32")
        assert arr.shape == self.shape and dtype == self.dtype, (
            f"{name}: Expected {self.shape} {self.dtype}, got {arr.shape} {dtype}")

    def zero_example(self):
        return np.zeros(self.shape, dtype=self.dtype)

    @property
    def row_bytes(self):
        return int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize

    @property
    def torch_dtype(self):
        return torch.from_numpy(np.zeros(1, dtype=self.dtype)).dtype


ReplayElement = collections.namedtuple("ReplayElement", ["name", "metadata"])


class ReplayBuffer:
    def __init__(
        self,
        stack_size: int = 1,
        replay_capacity: int = 10000,
        batch_size: int = 1,
        return_everything_as_stack: bool = False,
        return_as_timeline_format: bool = False,
        update_horizon: int = 1,
        gamma: float = 0.99,
        device=None,
    ) -> None:
        if replay_capacity < update_horizon + stack_size:
            raise ValueError(
                "There is not enough capacity to cover update_horizon and stack_size.")
        if return_as_timeline_format:
            raise NotImplementedError(
                "return_as_timeline_format (ragged python lists) is out of scope of reagent_b200")
        self._initialized_buffer = False
        self._stack_size = stack_size
        self._return_everything_as_stack = return_everything_as_stack
        self._return_as_timeline_format = return_as_timeline_format
        self._replay_capacity = replay_capacity
        self._batch_size = batch_size
        self._update_horizon = update_horizon
        self._gamma = gamma
        self._device = torch.device(device) if device is not None else None

        self.add_count = np.array(0)
        # gamma ** k as fp32, computed as the reference does (:367)
        self._decays = (self._gamma ** torch.arange(self._update_horizon)).unsqueeze(0)
        self._is_index_valid = torch.zeros(self._replay_capacity, dtype=torch.bool)
        self._num_valid_indices = 0
        self._num_transitions_in_current_episode = 0

        self._store: Dict[str, torch.Tensor] = {}
        self._storage_types: List[ReplayElement] = []
        self._batch_type = collections.namedtuple("filler", [])
        self._extra_keys: List[str] = []
        self._key_to_replay_elem: Dict[str, ReplayElement] = {}
        self._zero_transition = {}
        self._transition_elements = {}

        # device-side state
        self._terminal_host = np.zeros(self._replay_capacity, dtype=np.bool_)
        self._valid_dev = None
        self._valid_dirty: List[int] = []
        self._valid_index = None      # (counts, offsets) for uniform select
        self._valid_index_stale = True
        self._stage: Dict[str, torch.Tensor] = {}
        self._stage_n = 0
        self._stage_start = 0
        self._decays_dev = None
        # optional fused normalisation of `observation` (set_state_preprocessor)
        self._preproc = None
        # (B*A, A) identity tilings of sample_parametric_dqn_batch, per (B, A)
        self._tiled_eye_cache: Dict[tuple, torch.Tensor] = {}

    # ------------------------------------------------------------------ init
    def _dev(self):
        if self._device is None:
            if not torch.cuda.is_available():
                raise _lib.Rb200Error(
                    "reagent_b200.ReplayBuffer keeps its storage on the GPU and no CUDA device "
                    "is available (there is no CPU fallback)")
            self._device = torch.device("cuda", torch.cuda.current_device())
        return self._device

    def initialize_buffer(self, **kwargs):
        kwarg_keys = set(kwargs.keys())
        assert set(REQUIRED_KEYS).issubset(kwarg_keys), (
            f"{kwarg_keys} doesn't contain all of {REQUIRED_KEYS}")
        self._extra_keys = sorted(kwarg_keys - set(REQUIRED_KEYS))
        self._storage_types = [
            ReplayElement(k, DenseMetadata(k, kwargs[k])) for k in REQUIRED_KEYS + self._extra_keys]
        self._key_to_replay_elem = {e.name: e for e in self.get_storage_signature()}
        rmd = self._key_to_replay_elem["reward"].metadata
        if rmd.dtype != np.float32 or rmd.shape != ():
            raise NotImplementedError(
                f"reward must be a float scalar (got {rmd.dtype} {rmd.shape}); pass float rewards")
        self._create_storage()
        self._transition_elements = self.get_transition_elements()
        self._batch_type = collections.namedtuple("batch_type", self._transition_elements)
        self._zero_transition = {e.name: e.metadata.zero_example() for e in self._storage_types}
        self._initialized_buffer = True

    def _create_storage(self) -> None:
        dev = self._dev()
        for e in self.get_storage_signature():
            md = e.metadata
            shape = [self._replay_capacity, *md.shape]
            self._store[e.name] = torch.zeros(shape, dtype=md.torch_dtype, device=dev)
            self._stage[e.name] = torch.zeros([_STAGE_ROWS, *md.shape], dtype=md.torch_dtype)
            if torch.cuda.is_available():
                self._stage[e.name] = self._stage[e.name].pin_memory()
        self._valid_dev = torch.zeros(self._replay_capacity, dtype=torch.uint8, device=dev)
        self._decays_dev = self._decays.reshape(-1).to(dev).contiguous()

    @property
    def size(self) -> int:
        return self._num_valid_indices

    def set_index_valid_status(self, idx: int, is_valid: bool):
        old_valid = bool(self._is_index_valid[idx])
        if not old_valid and is_valid:
            self._num_valid_indices += 1
        elif old_valid and not is_valid:
            self._num_valid_indices -= 1
        assert self._num_valid_indices >= 0, f"{self._num_valid_indices} is negative"
        if old_valid != bool(is_valid):
            self._is_index_valid[idx] = is_valid
            self._valid_dirty.append(int(idx))
            self._valid_index_stale = True
            self._on_validity_change(int(idx), bool(is_valid))

    def _on_validity_change(self, idx: int, is_valid: bool):
        pass

    def get_add_args_signature(self) -> List[ReplayElement]:
        return self.get_storage_signature()

    def get_storage_signature(self) -> List[ReplayElement]:
        return self._storage_types

    def _add_zero_transition(self) -> None:
        self._add(**self._zero_transition)

    # ------------------------------------------------------------------- add
    def add(self, **kwargs):
        """circular_replay_buffer.py:468-522, verbatim semantics."""
        if not self._initialized_buffer:
            self.initialize_buffer(**kwargs)
        self._check_add_types(**kwargs)
        last_idx = (self.cursor() - 1) % self._replay_capacity
        if self.is_empty() or self._terminal_host[last_idx]:
            self._num_transitions_in_current_episode = 0
            for _ in range(self._stack_size - 1):
                self._add_zero_transition()
        cur_idx = self.cursor()
        self.set_index_valid_status(idx=cur_idx, is_valid=False)
        if self._num_transitions_in_current_episode >= self._update_horizon:
            idx = (cur_idx - self._update_horizon) % self._replay_capacity
            self.set_index_valid_status(idx=idx, is_valid=True)
        self._add(**kwargs)
        self._num_transitions_in_current_episode += 1
        for i in range(self._stack_size - 1):
            idx = (self.cursor() + i) % self._replay_capacity
            self.set_index_valid_status(idx=idx, is_valid=False)
        if kwargs["terminal"]:
            num_back = min(self._num_transitions_in_current_episode, self._update_horizon)
            for i in range(0, num_back):
                idx = (cur_idx - i) % self._replay_capacity
                self.set_index_valid_status(idx=idx, is_valid=True)

    def _add(self, **kwargs):
        self._check_args_length(**kwargs)
        self._add_transition(kwargs)

    def _add_transition(self, transition) -> None:
        cursor = self.cursor()
        if self._stage_n == min(_STAGE_ROWS, self._replay_capacity):
            self._flush()
        if self._stage_n == 0:
            self._stage_start = cursor
        row = self._stage_n
        for arg_name, value in transition.items():
            md = self._key_to_replay_elem[arg_name].metadata
            self._stage[arg_name][row] = torch.from_numpy(np.array(value, dtype=md.dtype))
        self._terminal_host[cursor] = bool(transition["terminal"])
        self._stage_n += 1
        self.add_count += 1

    def _flush(self):
        """Move staged transitions and validity changes to the device."""
        if not self._initialized_buffer:
            return
        dev = self._dev()
        n = self._stage_n
        if n > 0:
            cap = self._replay_capacity
            c0 = self._stage_start
            first = min(n, cap - c0)
            for k, st in self._stage.items():
                self._store[k][c0:c0 + first].copy_(st[:first], non_blocking=True)
                if first < n:
                    self._store[k][0:n - first].copy_(st[first:n], non_blocking=True)
            # the pinned staging rows are reused by the next add(): wait for the copies
            torch.cuda.current_stream().synchronize()
            self._stage_n = 0
        if self._valid_dirty:
            idx = np.unique(np.asarray(self._valid_dirty, dtype=np.int64))
            self._valid_dirty = []
            vals = self._is_index_valid[torch.from_numpy(idx)].to(torch.uint8)
            self._valid_dev[torch.from_numpy(idx).to(dev)] = vals.to(dev)

    def add_batch(self, **arrays):
        """N consecutive add() calls at once (identical end state), for bulk loading:
        every value is an array with a leading dimension N.  stack_size == 1 only."""
        n = len(arrays["terminal"])
        if self._stack_size != 1:
            for t in range(n):
                self.add(**{k: v[t] for k, v in arrays.items()})
            return
        if not self._initialized_buffer:
            self.initialize_buffer(**{k: np.asarray(v)[0] for k, v in arrays.items()})
        self._flush()
        cap = self._replay_capacity
        term = np.ascontiguousarray(np.asarray(arrays["terminal"]).astype(np.uint8))
        valid = self._is_index_valid.numpy().view(np.uint8)
        tstore = self._terminal_host.view(np.uint8)
        state = np.array([int(self.add_count), self._num_transitions_in_current_episode,
                          self._num_valid_indices], dtype=np.int64)
        start = int(self.add_count)
        self._pre_add_batch(start, n, arrays)
        _lib.lib().rb200_replay_add_batch_host(term.ctypes.data, n, cap, self._update_horizon,
                                               valid.ctypes.data, tstore.ctypes.data,
                                               state.ctypes.data)
        self.add_count = np.array(int(state[0]))
        self._num_transitions_in_current_episode = int(state[1])
        self._num_valid_indices = int(state[2])
        pos = (start + np.arange(n, dtype=np.int64)) % cap
        if n > cap:  # only the last `cap` rows survive
            keep = np.arange(n - cap, n)
        else:
            keep = np.arange(n)
        pos_t = torch.from_numpy(pos[keep]).to(self._dev())
        for e in self.get_add_args_signature():
            k = e.name
            if k not in arrays:
                continue
            md = e.metadata
            a = np.asarray(arrays[k])
            if a.dtype != md.dtype:
                a = a.astype(md.dtype)
            self._store[k][pos_t] = torch.from_numpy(np.ascontiguousarray(a[keep])).to(self._dev())
        self._valid_dev.copy_(torch.from_numpy(valid.copy()))
        self._valid_dirty = []
        self._valid_index_stale = True
        self._post_add_batch()

    def _pre_add_batch(self, start, n, arrays):
        pass

    def _post_add_batch(self):
        pass

    def _check_args_length(self, **kwargs):
        if len(kwargs) != len(self.get_add_args_signature()):
            raise ValueError(
                f"Add expects: {self.get_add_args_signature()}; received {kwargs}")

    def _check_add_types(self, **kwargs):
        self._check_args_length(**kwargs)
        for store_element in self.get_add_args_signature():
            store_element.metadata.validate(store_element.name, kwargs[store_element.name])

    def is_empty(self) -> bool:
        return self.add_count == 0

    def is_full(self) -> bool:
        return self.add_count >= self._replay_capacity

    def cursor(self) -> int:
        return int(self.add_count % self._replay_capacity)

    def is_valid_transition(self, index):
        return self._is_index_valid[index]

    # -------------------------------------------------------------- sampling
    def set_state_preprocessor(self, preprocessor):
        """Fuse a reagent_b200 Preprocessor (all features present) into the gather of
        `state` / `next_state` (north star: on-the-fly feature normalisation)."""
        self._preproc = preprocessor

    def _ensure_valid_index(self):
        if self._valid_index is None:
            nblk = (self._replay_capacity + _lib.VALID_BLOCK - 1) // _lib.VALID_BLOCK
            dev = self._dev()
            self._valid_index = (torch.zeros(nblk, dtype=torch.int32, device=dev),
                                 torch.zeros(nblk + 1, dtype=torch.int32, device=dev))
            self._valid_index_stale = True
        if self._valid_index_stale:
            counts, offsets = self._valid_index
            rc = _lib.lib().rb200_valid_index_build(
                self._valid_dev.data_ptr(), self._replay_capacity, counts.data_ptr(),
                offsets.data_ptr(), _lib.cur_stream())
            _lib.check(rc, "rb200_valid_index_build")
            self._valid_index_stale = False
        return self._valid_index

    def _index_source(self, args, batch_size, keep, ranks_dev=None):
        """Fill the index-selection part of the kernel arguments (uniform sampling:
        circular_replay_buffer.py:589-603).  `ranks_dev`: pre-uploaded torch.randint draws."""
        if self._num_valid_indices == 0:
            raise RuntimeError(
                f"Cannot sample {batch_size} since there are no valid indices so far.")
        counts, offsets = self._ensure_valid_index()
        if ranks_dev is None:
            ranks = torch.randint(self._num_valid_indices, (batch_size,))
            if torch.cuda.is_available():
                ranks = ranks.pin_memory()
            keep.append(ranks)
            ranks_d = ranks.to(self._dev(), non_blocking=True)
        else:
            ranks_d = ranks_dev
        keep.append(ranks_d)
        args.mode = _lib.SAMPLE_UNIFORM
        args.ranks = ranks_d.data_ptr()
        args.valid = self._valid_dev.data_ptr()
        args.valid_block_offsets = offsets.data_ptr()
        args.n_valid_blocks = counts.shape[0]

    def sample_index_batch(self, batch_size: int) -> torch.Tensor:
        """Returns a batch of valid indices sampled uniformly (device int64 tensor)."""
        self._flush()
        args = _lib.SampleArgsT()
        keep = []
        self._index_source(args, batch_size, keep)
        out = torch.empty(batch_size, dtype=torch.int64, device=self._dev())
        self._common_args(args, batch_size)
        args.indices_out = out.data_ptr()
        _lib.check(_lib.lib().rb200_replay_sample(args, _lib.cur_stream()), "rb200_replay_sample")
        return out

    def sample_all_valid_transitions(self):
        valid_indices = self._is_index_valid.nonzero().squeeze(1)
        assert valid_indices.ndim == 1
        return self.sample_transition_batch(batch_size=len(valid_indices), indices=valid_indices)

    def _common_args(self, args, batch_size):
        args.batch = batch_size
        args.capacity = self._replay_capacity
        args.update_horizon = self._update_horizon
        args.timeline_next = 0
        args.terminal = self._store["terminal"].data_ptr()
        args.reward = self._store["reward"].data_ptr()
        args.decays = self._decays_dev.data_ptr()

    def _stack_gather(self, key, idx_dev):
        """_get_stack_for_indices for stack_size > 1 (circular_replay_buffer.py:749-757):
        device index arithmetic + gather (cold path)."""
        stack_indices = idx_dev.unsqueeze(1) + torch.arange(-self._stack_size + 1, 1,
                                                            device=idx_dev.device)
        stack_indices %= self._replay_capacity
        sample = self._store[key][stack_indices]
        nd = len(self._key_to_replay_elem[key].metadata.shape)
        perm = [0] + list(range(2, nd + 2)) + [1]
        return sample.permute(*perm)

    def sample_transition_batch(self, batch_size=None, indices=None):
        """circular_replay_buffer.py:614-706.  Returns the namedtuple of DEVICE tensors in the
        reference's field order; 1-D results are (batch_size, 1)."""
        if batch_size is None:
            batch_size = self._batch_size
        self._flush()
        dev = self._dev()
        B = batch_size
        args = _lib.SampleArgsT()
        keep = []
        if indices is None:
            self._index_source(args, B, keep)
        else:
            assert isinstance(indices, torch.Tensor), (
                f"Indices {indices} have type {type(indices)} instead of torch.Tensor")
            ind = indices.to(device=dev, dtype=torch.int64).contiguous()
            assert len(ind) == B
            keep.append(ind)
            args.mode = _lib.SAMPLE_GIVEN
            args.indices_in = ind.data_ptr()
        self._common_args(args, B)
        out = {}
        out["indices"] = torch.empty(B, dtype=torch.int64, device=dev)
        out["step"] = torch.empty(B, dtype=torch.int64, device=dev)
        out["reward"] = torch.empty(B, dtype=torch.float32, device=dev)
        term_u8 = torch.empty(B, dtype=torch.uint8, device=dev)
        args.indices_out = out["indices"].data_ptr()
        args.step_out = out["step"].data_ptr()
        args.reward_out = out["reward"].data_ptr()
        args.terminal_out = term_u8.data_ptr()
        self._extra_outputs(args, B, out, keep)

        simple = self._stack_size == 1
        specs = []
        obs_md = self._key_to_replay_elem["observation"].metadata
        fused_obs = simple and obs_md.dtype == np.float32 and len(obs_md.shape) == 1
        if fused_obs:
            S = obs_md.shape[0]
            args.obs = self._store["observation"].data_ptr()
            args.obs_dim = S
            s_out = S
            if self._preproc is not None:
                cols, quant, s_out = self._preproc.device_program(dev)
                args.cols = cols.data_ptr()
                args.quantiles = quant.data_ptr()
                keep += [cols, quant]
            args.obs_out_dim = s_out
            out["state"] = torch.empty(B, s_out, dtype=torch.float32, device=dev)
            out["next_state"] = torch.empty(B, s_out, dtype=torch.float32, device=dev)
            args.state = out["state"].data_ptr()
            args.next_state = out["next_state"].data_ptr()
        for name in self._transition_elements:
            if name in out or name in ("terminal", "sampling_probabilities"):
                continue
            if name == "state":
                key, which = "observation", 0
            elif name == "next_state":
                key, which = "observation", 1
            elif name in self._store:
                key, which = name, 0
            elif name.startswith("next_") and name[len("next_"):] in self._store:
                key, which = name[len("next_"):], 1
            else:
                out[name] = None
                continue
            if name == "reward":
                continue
            md = self._key_to_replay_elem[key].metadata
            if simple:
                t = torch.empty([B, *md.shape], dtype=md.torch_dtype, device=dev)
                out[name] = t
                specs.append((self._store[key], t, md.row_bytes, which))
            else:
                out[name] = (key, which)  # resolved after the kernel with the indices
        if self._return_everything_as_stack and simple:
            md = self._key_to_replay_elem["reward"].metadata
            t = torch.empty([B, *md.shape], dtype=md.torch_dtype, device=dev)
            specs.append((self._store["reward"], t, md.row_bytes, 0))
            out["reward"] = t
        if len(specs) > _lib.MAX_GATHER_SPECS:
            raise NotImplementedError(
                f"more than {_lib.MAX_GATHER_SPECS} dense replay elements per launch")
        args.n_specs = len(specs)
        for i, (src, dst, rb, which) in enumerate(specs):
            args.specs[i].src = src.data_ptr()
            args.specs[i].dst = dst.data_ptr()
            args.specs[i].row_bytes = rb
            args.specs[i].which = which
        _lib.check(_lib.lib().rb200_replay_sample(args, _lib.cur_stream()), "rb200_replay_sample")

        out["terminal"] = term_u8.to(torch.bool)
        if not simple:
            idx = out["indices"]
            nxt = (idx + out["step"]) % self._replay_capacity
            for name, v in list(out.items()):
                if isinstance(v, tuple):
                    key, which = v
                    res = self._stack_gather(key, nxt if which else idx)
                    out[name] = res
            if self._return_everything_as_stack:
                out["reward"] = self._stack_gather("reward", idx)
        batch_arrays = []
        for name in self._transition_elements:
            t = out.get(name)
            if isinstance(t, torch.Tensor) and t.ndim == 1:
                t = t.unsqueeze(1)
            batch_arrays.append(t)
        return self._batch_type(*batch_arrays)

    def _extra_outputs(self, args, B, out, keep):
        """Hook for subclasses (prioritized: sampling probabilities)."""
        pass

    # ---------------------------------------------------- fused trainer batches
    # ---- caller-owned output buffers for the fused trainer batches -----------------------
    _out_pool = None

    def output_buffers(self, pool: dict):
        """Context manager: while active, the fused `sample_*_batch` calls write their outputs
        into the tensors of `pool` (filled on first use) instead of fresh allocations, so a
        captured sampling launch can feed another captured graph through fixed addresses
        (training/fused_step.py, prefetch mode)."""
        import contextlib

        @contextlib.contextmanager
        def cm():
            prev, self._out_pool = self._out_pool, pool
            try:
                yield pool
            finally:
                self._out_pool = prev
        return cm()

    def _alloc(self, name, *shape, dtype=torch.float32):
        pool = self._out_pool
        if pool is None:
            return torch.empty(*shape, dtype=dtype, device=self._dev())
        t = pool.get(name)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = torch.empty(*shape, dtype=dtype, device=self._dev())
            pool[name] = t
        return t

    def _fused_common(self, batch_size, indices, index_kwargs):
        if self._stack_size != 1:
            raise NotImplementedError("fused trainer batches need stack_size == 1")
        obs_md = self._key_to_replay_elem["observation"].metadata
        if obs_md.dtype != np.float32 or len(obs_md.shape) != 1:
            raise NotImplementedError("fused trainer batches need a flat float32 observation")
        self._flush()
        dev = self._dev()
        B = batch_size
        args = _lib.SampleArgsT()
        keep = []
        if indices is None:
            self._index_source(args, B, keep, **index_kwargs)
        else:
            ind = indices.to(device=dev, dtype=torch.int64).contiguous()
            keep.append(ind)
            args.mode = _lib.SAMPLE_GIVEN
            args.indices_in = ind.data_ptr()
        self._common_args(args, B)
        S = obs_md.shape[0]
        args.obs = self._store["observation"].data_ptr()
        args.obs_dim = S
        s_out = S
        if self._preproc is not None:
            cols, quant, s_out = self._preproc.device_program(dev)
            args.cols = cols.data_ptr()
            args.quantiles = quant.data_ptr()
            keep += [cols, quant]
        args.obs_out_dim = s_out
        t = {
            "state": self._alloc("state", B, s_out),
            "next_state": self._alloc("next_state", B, s_out),
            "reward": self._alloc("reward", B, 1),
            "not_terminal": self._alloc("not_terminal", B, 1),
            "step": self._alloc("step", B, 1),
            "indices": self._alloc("indices", B, 1, dtype=torch.int64),
        }
        args.state = t["state"].data_ptr()
        args.next_state = t["next_state"].data_ptr()
        args.reward_out = t["reward"].data_ptr()
        args.not_terminal_out = t["not_terminal"].data_ptr()
        args.step_f32_out = t["step"].data_ptr()
        args.indices_out = t["indices"].data_ptr()
        extra = {}
        self._extra_outputs(args, B, extra, keep)
        for k, v in extra.items():
            t[k] = v.unsqueeze(1) if v.ndim == 1 else v
        return args, t, keep

    def _ones(self, B, A):
        key = (B, A)
        c = getattr(self, "_ones_cache", None)
        if c is None or c[0] != key:
            self._ones_cache = (key, torch.ones(B, A, device=self._dev()))
        return self._ones_cache[1]

    def _tiled_eye(self, B, A):
        """get_possible_actions_for_gym (trainer_preprocessor.py:357-367): the (B*A, A) tiling of
        the A x A identity, one cached device constant per shape, so a sampling launch that
        returns it can be captured into a CUDA graph."""
        # never evicted: a captured graph keeps reading the constant of its shape, and a
        # workload samples a handful of (batch size, action count) shapes
        t = self._tiled_eye_cache.get((B, A))
        if t is None:
            t = torch.eye(A, device=self._dev()).repeat(B, 1)
            self._tiled_eye_cache[(B, A)] = t
        return t

    def _sample_onehot(self, batch_size, num_actions, indices, index_kwargs, stored_masks):
        """The ONE rb200_replay_sample launch behind the discrete-action batches: state,
        next state, reward, not_terminal, the one-hot action and next action (zeroed on
        terminal rows, one_hot_actions of trainer_preprocessor.py:72-97), the stored `log_prob`
        and, with `stored_masks`, the stored `possible_actions_mask` and its next twin.
        Returns (tensors, action, next_action, action_probability | None, masks | None)."""
        amd = self._key_to_replay_elem["action"].metadata
        if amd.dtype != np.int64 or amd.shape != ():
            raise NotImplementedError("discrete batches need an int64 scalar action")
        args, t, keep = self._fused_common(batch_size, indices, index_kwargs)
        B = batch_size
        action = self._alloc("action", B, num_actions)
        next_action = self._alloc("next_action", B, num_actions)
        args.action_i64 = self._store["action"].data_ptr()
        args.num_actions = num_actions
        args.action_onehot = action.data_ptr()
        args.next_action_onehot = next_action.data_ptr()
        prob = None
        ns = 0

        def spec(key, name, which, width):
            nonlocal ns
            out = self._alloc(name, B, width)
            args.specs[ns].src = self._store[key].data_ptr()
            args.specs[ns].dst = out.data_ptr()
            args.specs[ns].row_bytes = 4 * width
            args.specs[ns].which = which
            ns += 1
            return out

        if "log_prob" in self._store:
            prob = spec("log_prob", "log_prob", 0, 1)
        masks = None
        if stored_masks and "possible_actions_mask" in self._store:
            md = self._key_to_replay_elem["possible_actions_mask"].metadata
            if md.dtype != np.float32 or md.shape != (num_actions,):
                raise NotImplementedError("possible_actions_mask must be float32 [num_actions]")
            masks = (spec("possible_actions_mask", "possible_actions_mask", 0, num_actions),
                     spec("possible_actions_mask", "possible_next_actions_mask", 1, num_actions))
        args.n_specs = ns
        _lib.check(_lib.lib().rb200_replay_sample(args, _lib.cur_stream()), "rb200_replay_sample")
        return t, action, next_action, None if prob is None else prob.exp(), masks

    def sample_discrete_dqn_batch(self, batch_size, num_actions, indices=None, **index_kwargs):
        """sample_transition_batch + DiscreteDqnInputMaker.__call__
        (gym/preprocessors/trainer_preprocessor.py:100-158) as ONE launch: returns an
        rlt.DiscreteDqnInput of device tensors (masks are ones, step carries the n-step
        length as float, time_diff None)."""
        from ..core import types as rlt

        t, action, next_action, prob, masks = self._sample_onehot(
            batch_size, num_actions, indices, index_kwargs, stored_masks=True)
        # DiscreteDqnInputMaker :131-139: masks come from the `possible_actions_mask` extra
        # (and its `next_` twin) when the buffer stores one, else ones
        pam, pnam = masks if masks is not None else (self._ones(batch_size, num_actions),) * 2
        batch = rlt.DiscreteDqnInput(
            state=rlt.FeatureData(t["state"]), next_state=rlt.FeatureData(t["next_state"]),
            reward=t["reward"], time_diff=None, step=t["step"], not_terminal=t["not_terminal"],
            action=action, next_action=next_action, possible_actions_mask=pam,
            possible_next_actions_mask=pnam, extras=rlt.ExtraData(action_probability=prob))
        batch.indices = t["indices"]
        batch.sampling_probabilities = t.get("sampling_probabilities")
        return batch

    def sample_parametric_dqn_batch(self, batch_size, num_actions, indices=None,
                                    **index_kwargs):
        """sample_transition_batch + ParametricDqnInputMaker.__call__
        (gym/preprocessors/trainer_preprocessor.py:370-413) as ONE launch: returns an
        rlt.ParametricDqnInput of device tensors.  The actions are one-hot FeatureData (the next
        action zeroed on terminal rows); the possible (next) actions are the (B*A, A) identity
        tiling and both masks are ones, cached device constants; step and time_diff are None,
        as the reference's input maker passes them.  A stored `possible_actions_mask` extra is
        ignored, as the reference ignores it."""
        from ..core import types as rlt

        t, action, next_action, prob, _ = self._sample_onehot(
            batch_size, num_actions, indices, index_kwargs, stored_masks=False)
        tiled = rlt.FeatureData(self._tiled_eye(batch_size, num_actions))
        ones = self._ones(batch_size, num_actions)
        batch = rlt.ParametricDqnInput(
            state=rlt.FeatureData(t["state"]), next_state=rlt.FeatureData(t["next_state"]),
            reward=t["reward"], time_diff=None, step=None, not_terminal=t["not_terminal"],
            action=rlt.FeatureData(action), next_action=rlt.FeatureData(next_action),
            possible_actions=tiled, possible_actions_mask=ones, possible_next_actions=tiled,
            possible_next_actions_mask=ones, extras=rlt.ExtraData(action_probability=prob))
        batch.indices = t["indices"]
        batch.sampling_probabilities = t.get("sampling_probabilities")
        return batch

    def _action_bounds(self, action_low, action_high, dev):
        """Device copies of the action range, cached per value: the host->device copy happens
        once, so a sampling launch with known bounds can be captured into a CUDA graph."""
        lo = np.ascontiguousarray(np.asarray(action_low, dtype=np.float32).reshape(-1))
        hi = np.ascontiguousarray(np.asarray(action_high, dtype=np.float32).reshape(-1))
        key = (lo.tobytes(), hi.tobytes(), str(dev))
        cache = self.__dict__.setdefault("_action_bounds_cache", {})
        out = cache.get(key)
        if out is None:
            if len(cache) >= 16:
                cache.clear()
            out = (torch.from_numpy(lo.copy()).to(dev), torch.from_numpy(hi.copy()).to(dev))
            cache[key] = out
        return out

    def sample_policy_network_batch(self, batch_size, action_low, action_high, indices=None,
                                    **index_kwargs):
        """sample_transition_batch + PolicyNetworkInputMaker.__call__
        (trainer_preprocessor.py:161-227) as ONE launch -> rlt.PolicyNetworkInput."""
        from ..core import types as rlt
        from ..core.parameters import CONTINUOUS_TRAINING_ACTION_RANGE

        amd = self._key_to_replay_elem["action"].metadata
        if amd.dtype != np.float32 or len(amd.shape) != 1:
            raise NotImplementedError("continuous batches need a flat float32 action")
        args, t, keep = self._fused_common(batch_size, indices, index_kwargs)
        B, dev, A = batch_size, self._dev(), amd.shape[0]
        lo, hi = self._action_bounds(action_low, action_high, dev)
        action = self._alloc("action", B, A)
        next_action = self._alloc("next_action", B, A)
        args.action_f32 = self._store["action"].data_ptr()
        args.action_dim = A
        args.action_rescaled = action.data_ptr()
        args.next_action_rescaled = next_action.data_ptr()
        args.action_low = lo.data_ptr()
        args.action_high = hi.data_ptr()
        args.train_low, args.train_high = CONTINUOUS_TRAINING_ACTION_RANGE
        prob = None
        if "log_prob" in self._store:  # extras.action_probability = log_prob.exp() (:206)
            prob = self._alloc("log_prob", B, 1)
            args.n_specs = 1
            args.specs[0].src = self._store["log_prob"].data_ptr()
            args.specs[0].dst = prob.data_ptr()
            args.specs[0].row_bytes = 4
            args.specs[0].which = 0
        _lib.check(_lib.lib().rb200_replay_sample(args, _lib.cur_stream()), "rb200_replay_sample")
        batch = rlt.PolicyNetworkInput(
            state=rlt.FeatureData(t["state"]), next_state=rlt.FeatureData(t["next_state"]),
            reward=t["reward"], time_diff=None, step=t["step"], not_terminal=t["not_terminal"],
            action=rlt.FeatureData(action), next_action=rlt.FeatureData(next_action),
            extras=rlt.ExtraData(action_probability=None if prob is None else prob.exp()))
        batch.indices = t["indices"]
        batch.sampling_probabilities = t.get("sampling_probabilities")
        return batch

    def get_transition_elements(self):
        extra_names = []
        for name in self._extra_keys:
            for prefix in ["", "next_"]:
                extra_names.append(f"{prefix}{name}")
        return ["state", "action", "reward", "next_state", "next_action", "next_reward",
                "terminal", "indices", "step", *extra_names]

    # ------------------------------------------------------------ checkpoint
    def _generate_filename(self, checkpoint_dir, name, suffix):
        return os.path.join(checkpoint_dir, "{}_ckpt.{}.gz".format(name, suffix))

    def _return_checkpointable_elements(self):
        checkpointable_elements = {}
        for member_name, member in self.__dict__.items():
            if member_name == "_store":
                for array_name, array in self._store.items():
                    checkpointable_elements[STORE_FILENAME_PREFIX + array_name] = array
            elif not member_name.startswith("_"):
                checkpointable_elements[member_name] = member
        return checkpointable_elements

    def save(self, checkpoint_dir, iteration_number):
        """Same files as the reference (:810-853): one gzip per public attribute and per
        `_store` array (np.save), keeping the last CHECKPOINT_DURATION iterations."""
        if not os.path.exists(checkpoint_dir):
            return
        self._flush()
        elems = self._return_checkpointable_elements()
        for attr in elems:
            filename = self._generate_filename(checkpoint_dir, attr, iteration_number)
            with open(filename, "wb") as f:
                with gzip.GzipFile(fileobj=f) as outfile:
                    if attr.startswith(STORE_FILENAME_PREFIX):
                        array_name = attr[len(STORE_FILENAME_PREFIX):]
                        np.save(outfile, self._store[array_name].cpu().numpy(), allow_pickle=False)
                    elif isinstance(self.__dict__[attr], np.ndarray):
                        np.save(outfile, self.__dict__[attr], allow_pickle=False)
                    else:
                        pickle.dump(self.__dict__[attr], outfile)
            stale = iteration_number - CHECKPOINT_DURATION
            if stale >= 0:
                try:
                    os.remove(self._generate_filename(checkpoint_dir, attr, stale))
                except FileNotFoundError:
                    pass

    def load(self, checkpoint_dir, suffix):
        if getattr(self, "_device_resident", None) is not None:
            raise RuntimeError("the buffer is device-resident: call DeviceReplay.sync_to_host() before load()")
        elems = self._return_checkpointable_elements()
        for attr in elems:
            filename = self._generate_filename(checkpoint_dir, attr, suffix)
            if not os.path.exists(filename):
                raise FileNotFoundError(None, None, "Missing file: {}".format(filename))
        for attr in elems:
            filename = self._generate_filename(checkpoint_dir, attr, suffix)
            with open(filename, "rb") as f:
                with gzip.GzipFile(fileobj=f) as infile:
                    if attr.startswith(STORE_FILENAME_PREFIX):
                        array_name = attr[len(STORE_FILENAME_PREFIX):]
                        arr = np.load(infile, allow_pickle=False)
                        self._store[array_name].copy_(torch.from_numpy(arr))
                        if array_name == "terminal":
                            self._terminal_host = arr.astype(np.bool_).reshape(-1).copy()
                    elif isinstance(self.__dict__[attr], np.ndarray):
                        self.__dict__[attr] = np.load(infile, allow_pickle=False)
                    else:
                        self.__dict__[attr] = pickle.load(infile)
        # The loaded arrays replace whatever was staged or mirrored on the device: drop the rows
        # still in the pinned staging block (the store they would be flushed into was just
        # overwritten) and rebuild the device-side validity / priority mirrors.
        self._stage_n = 0
        self._valid_dirty = []
        self._valid_index_stale = True
        if self._valid_dev is not None:
            self._valid_dev.copy_(self._is_index_valid.to(torch.uint8))
        self._post_add_batch()
