"""World-model evaluators (reagent/evaluation/world_model_evaluator.py): the loss of a batch, how
much the loss rises when one feature is replaced by its mean (feature importance), and how far
the predicted next-state means move when the actions are shuffled (feature sensitivity).

The reference runs one MDN-RNN forward per feature, each followed by a host read-back.  Here
the original batch and every perturbed copy are the variants of ONE rb200_mdnrnn_eval launch
(csrc/rb200_mdnrnn.cu), each variant's losses the bits MDNRNNTrainer.get_loss gives on that
copy; the fill values and the sensitivity reduction are one launch each, and every `evaluate`
reads back once.  The evaluators keep their own device buffers, so an evaluation leaves the
trainer's next update unchanged.
"""
import logging
from typing import Dict, List, Optional

import numpy as np
import torch

from .. import _lib
from ..core.types import MemoryNetworkInput

logger = logging.getLogger(__name__)

LOSS_KEYS = ("gmm", "bce", "mse", "loss")


def feature_groups(starts: List[int], dim: int, num: int, what: str):
    """[(begin, end)] of the `num` features whose first columns are `starts` in a vector of
    `dim` columns, feature i ending where i + 1 starts (the last at `dim`)."""
    starts = [int(s) for s in starts]
    if len(starts) != num:
        raise ValueError(f"{what}: {len(starts)} feature start indices for {num} features")
    bounds = starts + [int(dim)]
    if not starts or starts[0] != 0 or any(b <= a for a, b in zip(bounds, bounds[1:])):
        raise ValueError(f"{what}: feature start indices {starts} must start at 0, increase "
                         f"strictly and stay below the dimension {dim}")
    return list(zip(bounds[:-1], bounds[1:]))


def importance_variants(discrete_action: bool, action_dim: int, state_dim: int,
                        action_groups, state_groups):
    """The variant table of feature importance: [(col_begin, col_end, fill_off)] over the
    columns of x = cat(action, state), variant 0 the original batch, then one per action
    feature and one per state feature; and the fill layout (n_eye, groups): the fill buffer
    holds n_eye floats of the discrete actions' one-hots (row i = e_i), then one value per
    column of x for the feature groups `groups` (x columns) that get a mean / median fill."""
    A = action_dim
    rows = [(0, 0, 0)]
    if discrete_action:
        n_eye = A * A
        rows += [(0, A, i * A) for i in range(A)]
        groups = []
    else:
        n_eye = 0
        rows += [(b, e, b) for b, e in action_groups]
        groups = list(action_groups)
    rows += [(A + b, A + e, n_eye + A + b) for b, e in state_groups]
    groups += [(A + b, A + e) for b, e in state_groups]
    return rows, n_eye, groups


def _features(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise _lib.Rb200Error(f"world-model evaluation: {name} must be a CUDA tensor "
                              "(reagent_b200 runs on CUDA only; there is no CPU path)")
    if t.dim() != 3:
        raise ValueError(f"world-model evaluation: {name} must be [T, B, dim], got "
                         f"{tuple(t.shape)}")
    return t.float().contiguous()


def _targets(batch: MemoryNetworkInput, T: int, B: int, S: int):
    ns = _features(batch.next_state.float_features, "next_state")
    out = [ns]
    for name in ("reward", "not_terminal"):
        t = getattr(batch, name)
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise _lib.Rb200Error(f"world-model evaluation: {name} must be a CUDA tensor")
        out.append(t.float().reshape(T, B).contiguous() if t.numel() == T * B else t)
    if tuple(ns.shape) != (T, B, S) or any(t.numel() != T * B for t in out[1:]):
        raise ValueError(f"world-model evaluation: next_state {tuple(ns.shape)}, reward and "
                         f"not_terminal must cover [T, B] = [{T}, {B}]")
    return out


def _group_array(groups):
    g = [0] * (_lib.MDNRNN_MAX_INPUT + 1)
    for i, (b, _) in enumerate(groups):
        g[i] = b
    g[len(groups)] = groups[-1][1]
    return g


class _EvalBuffers:
    """Device buffers of one (T, B, variants) shape of one evaluator."""

    def __init__(self, T, B, V, n_fill, mus_floats, device):
        n_blocks = -(-B // _lib.MDNRNN_ROWS_PER_BLOCK)
        self.key = (T, B, V, n_fill, mus_floats, device)
        self.loss_partials = torch.zeros(V * 3 * n_blocks, device=device)
        self.counter = torch.zeros(V, dtype=torch.int32, device=device)
        self.loss = torch.zeros(V, 4, device=device)
        self.fill = torch.zeros(max(n_fill, 1), device=device)
        self.mus = torch.empty(mus_floats, device=device) if mus_floats else None


class _WorldModelEval:
    """What the three evaluators share: the trainer's network and loss settings, and one
    rb200_mdnrnn_eval launch over a variant table."""

    def __init__(self, trainer):
        self.trainer = trainer
        self._bufs: Optional[_EvalBuffers] = None

    @property
    def _net(self):
        return self.trainer.memory_network.mdnrnn

    def _inputs(self, batch: MemoryNetworkInput):
        if not isinstance(batch, MemoryNetworkInput):
            raise TypeError(f"world-model evaluation needs a MemoryNetworkInput, got "
                            f"{type(batch).__name__}")
        state = _features(batch.state.float_features, "state")
        action = _features(batch.action.float_features, "action")
        T, B, S = state.shape
        net = self._net
        if S != net.state_dim or tuple(action.shape) != (T, B, net.action_dim):
            raise ValueError(f"world-model evaluation: state {tuple(state.shape)} and action "
                             f"{tuple(action.shape)} do not fit the network (state_dim "
                             f"{net.state_dim}, action_dim {net.action_dim})")
        _lib.require_current_device(state.device)
        return state, action, _targets(batch, T, B, S)

    def _buffers(self, T, B, V, n_fill, mus_floats, device) -> _EvalBuffers:
        key = (T, B, V, n_fill, mus_floats, device)
        if self._bufs is None or self._bufs.key != key:
            self._bufs = _EvalBuffers(T, B, V, n_fill, mus_floats, device)
        return self._bufs

    def _launch(self, state, action, targets, variants, ws: _EvalBuffers, perm=None,
                perm_variant=-1, with_mus=False, gmm_state_dim=None):
        """rb200_mdnrnn_eval over `variants` [(col_begin, col_end, fill_off)]; losses into
        ws.loss [V, 4] with loss = gmm / (state_dim + 2) + bce + mse, as get_loss(batch,
        state_dim) computes it; state_dim is gmm_state_dim, or the batch's without it."""
        T, B, S = state.shape
        p = self.trainer.params
        e = _lib.MdnrnnEvalArgsT()
        e.net = self._net.args(T, B)
        a = e.net
        ns, r, nt = targets
        a.state, a.action = state.data_ptr(), action.data_ptr()
        a.next_state, a.reward, a.not_terminal = ns.data_ptr(), r.data_ptr(), nt.data_ptr()
        a.next_state_weight = p.next_state_loss_weight
        a.not_terminal_weight = p.not_terminal_loss_weight
        a.reward_weight = p.reward_loss_weight
        a.gmm_divisor = float((S if gmm_state_dim is None else gmm_state_dim) + 2)
        a.fit_only_one_next_step = int(p.fit_only_one_next_step)
        e.num_variants = len(variants)
        for v, (c0, c1, off) in enumerate(variants):
            e.col_begin[v], e.col_end[v], e.fill_off[v] = c0, c1, off
        e.fill, e.fill_len = ws.fill.data_ptr(), ws.fill.numel()
        e.perm_variant = perm_variant
        e.perm = perm.data_ptr() if perm is not None else None
        e.mus = ws.mus.data_ptr() if with_mus else None
        e.loss_partials, e.tile_counter = ws.loss_partials.data_ptr(), ws.counter.data_ptr()
        e.loss = ws.loss.data_ptr()
        _lib.check(_lib.lib().rb200_mdnrnn_eval(e, _lib.cur_stream()), "rb200_mdnrnn_eval")


class LossEvaluator(_WorldModelEval):
    """The four losses of a batch, as host floats: get_loss(batch, state_dim) of the trainer,
    so loss = gmm / (state_dim + 2) + bce + mse with the constructor's state_dim."""

    def __init__(self, trainer, state_dim: int) -> None:
        super().__init__(trainer)
        self.state_dim = state_dim

    def evaluate(self, tdp: MemoryNetworkInput) -> Dict[str, float]:
        self._net.eval()
        state, action, targets = self._inputs(tdp)
        T, B, _ = state.shape
        ws = self._buffers(T, B, 1, 0, 0, state.device)
        self._launch(state, action, targets, [(0, 0, 0)], ws, gmm_state_dim=self.state_dim)
        vals = ws.loss[0].cpu().tolist()
        self._net.train()
        out = dict(zip(LOSS_KEYS, vals))
        return {k: out[k] for k in ("loss", "gmm", "bce", "mse")}


class FeatureImportanceEvaluator(_WorldModelEval):
    """Per feature, the rise of the trainer's loss when that feature is replaced by its
    average over the batch: actions first, then states."""

    def __init__(self, trainer, discrete_action: bool, state_feature_num: int,
                 action_feature_num: int, sorted_action_feature_start_indices: List[int],
                 sorted_state_feature_start_indices: List[int]) -> None:
        """A feature is a run of columns: feature i of the action (state) vector spans from
        its entry in sorted_action_feature_start_indices (sorted_state_feature_start_indices)
        to the next entry, the last one to the end of the vector, so a one-hot enum is one
        feature.  With discrete_action, action i is the one-hot column i instead."""
        super().__init__(trainer)
        self.discrete_action = discrete_action
        self.state_feature_num = state_feature_num
        self.action_feature_num = action_feature_num
        self.sorted_action_feature_start_indices = sorted_action_feature_start_indices
        self.sorted_state_feature_start_indices = sorted_state_feature_start_indices

    def variants(self, action_dim: int, state_dim: int):
        """(variant table, n_eye, fill groups) of importance_variants for these dimensions."""
        if self.discrete_action:
            assert action_dim == self.action_feature_num
            action_groups = None
        else:
            action_groups = feature_groups(self.sorted_action_feature_start_indices, action_dim,
                                           self.action_feature_num, "action features")
        state_groups = feature_groups(self.sorted_state_feature_start_indices, state_dim,
                                      self.state_feature_num, "state features")
        return importance_variants(self.discrete_action, action_dim, state_dim, action_groups,
                                   state_groups)

    def evaluate(self, batch: MemoryNetworkInput):
        """{"feature_loss_increase": float32 [action features + state features]}: for each
        feature, loss(batch with the feature replaced at every step and row) - loss(batch).
        A one-column feature is replaced by its mean, a wider one by the one-hot at the first
        column whose count is the lower median of its columns' counts, and with
        discrete_action action i by e_i.  The targets are never changed."""
        self._net.eval()
        state, action, targets = self._inputs(batch)
        T, B, S = state.shape
        A = action.shape[2]
        variants, n_eye, groups = self.variants(A, S)
        ws = self._buffers(T, B, len(variants), n_eye + A + S, 0, state.device)
        if n_eye:
            ws.fill[:n_eye].copy_(torch.eye(A, device=state.device).reshape(-1))
        f = _lib.MdnrnnFillArgsT()
        f.rows, f.action_dim, f.state_dim = T * B, A, S
        f.action, f.state = action.data_ptr(), state.data_ptr()
        f.num_groups = len(groups)
        f.group_begin[:] = _group_array(groups)
        f.fill = ws.fill.data_ptr() + 4 * n_eye
        st = _lib.cur_stream()
        _lib.check(_lib.lib().rb200_mdnrnn_fill_values(f, st), "rb200_mdnrnn_fill_values")
        self._launch(state, action, targets, variants, ws)
        # loss_v - loss_0 in fp32: the reference's fp64 difference of two fp32 losses, stored
        # into an fp32 tensor, is the same correctly rounded difference
        feature_importance = (ws.loss[1:, 3] - ws.loss[0, 3]).cpu()
        self._net.train()
        logger.info("world model: loss increase per feature %s", feature_importance.tolist())
        return {"feature_loss_increase": feature_importance.numpy()}

    def fill_values(self) -> torch.Tensor:
        """The fill buffer of the last `evaluate`: the one-hots of discrete actions, then
        each feature group's mean or median one-hot at its columns of x (a device view)."""
        return self._bufs.fill


class FeatureSensitivityEvaluator(_WorldModelEval):
    """Per state feature, how far the predicted next-state means move when the actions are
    shuffled across the batch."""

    def __init__(self, trainer, state_feature_num: int,
                 sorted_state_feature_start_indices: List[int]) -> None:
        super().__init__(trainer)
        self.state_feature_num = state_feature_num
        self.sorted_state_feature_start_indices = sorted_state_feature_start_indices

    def evaluate(self, batch: MemoryNetworkInput, perm: Optional[torch.Tensor] = None):
        """{"feature_sensitivity": float32 [state features]}: the mean over (T, B, G) of the
        sum over the feature's columns of |mus(shuffled actions) - mus(actions)|, where row b
        takes the actions of row perm[b] at every step.  `perm` defaults to torch.randperm(B)
        from torch's CPU generator, as the reference draws it; pass a recorded one to repeat
        an evaluation."""
        assert isinstance(batch, MemoryNetworkInput)
        self._net.eval()
        state, action, targets = self._inputs(batch)
        T, B, S = state.shape
        groups = feature_groups(self.sorted_state_feature_start_indices, S,
                                self.state_feature_num, "state features")
        if perm is None:
            perm = torch.randperm(B)
        perm = torch.as_tensor(perm)
        if perm.is_cuda:
            perm = perm.cpu()
        perm = perm.to(torch.int64).reshape(-1)
        if perm.numel() != B or (B and (int(perm.min()) < 0 or int(perm.max()) >= B)):
            raise ValueError(f"FeatureSensitivityEvaluator: perm must hold {B} indices in "
                             f"[0, {B})")
        net = self._net
        G = net.num_gaussians
        n_mus = T * B * G * S
        ws = self._buffers(T, B, 2, 0, 2 * n_mus, state.device)
        # from pinned memory, so that the upload does not wait for the stream: the read-back
        # below is this call's only host synchronisation
        perm_dev = perm.pin_memory().to(state.device, non_blocking=True)
        self._launch(state, action, targets, [(0, 0, 0), (0, 0, 0)], ws, perm=perm_dev,
                     perm_variant=1, with_mus=True)
        out = torch.empty(len(groups), device=state.device)
        f = _lib.MdnrnnSensitivityArgsT()
        f.rows, f.state_dim, f.gaussians = T * B, S, G
        f.mus0, f.mus1 = ws.mus.data_ptr(), ws.mus.data_ptr() + 4 * n_mus
        f.num_groups = len(groups)
        f.group_begin[:] = _group_array(groups)
        f.out = out.data_ptr()
        _lib.check(_lib.lib().rb200_mdnrnn_sensitivity(f, _lib.cur_stream()),
                   "rb200_mdnrnn_sensitivity")
        feature_sensitivity = out.cpu()
        net.train()
        logger.info("world model: sensitivity per state feature %s", feature_sensitivity.tolist())
        return {"feature_sensitivity": feature_sensitivity.numpy()}

    def means(self) -> torch.Tensor:
        """The predicted next-state means of the last `evaluate`, [2, T, B, G, S]: the
        original batch's, then the shuffled actions' (a device view)."""
        ws = self._bufs
        T, B = ws.key[0], ws.key[1]
        net = self._net
        return ws.mus.view(2, T, B, net.num_gaussians, net.state_dim)
