"""SlateQTrainer (reagent/training/slate_q_trainer.py:34-276) on the generic kernels of this
library.  q_network(state, doc) is the critic-shaped MLP of ParametricDQN.  Per update:

  * the target network scores EVERY next-state candidate in one rb200_mlp_forward_tiled launch
    (the tiled next state is built per row tile and never written to HBM);
  * rb200_slateq_head picks the next slate from those scores -- next_action (SARSA) or the
    top slate_size of q_target * docs_value (max-Q, TOP_K) -- weights it by the docs value,
    forms the target and writes the MSE loss and d loss / d q;
  * the current slate's input cat(state.repeat_interleave(K), docs[b, action]) is materialised
    once (the first layer's weight gradient reads it), run through rb200_mlp_forward with saved
    activations, then rb200_mlp_backward + rb200_mlp_wgrad, FusedAdam and SoftUpdate.

An index of action / next_action outside [-C, C) -- the reference's IndexError -- is flagged by
the head on the device.  The trainer raises IndexError for it at the start of a later update,
once the flag's copy to the host has landed, or at once from raise_if_failed(), which
synchronises."""
import enum
from typing import Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import (EvaluationParameters, RLParameters, SlateOptMethod,
                               SlateOptParameters)
from ..models.arena import run_mlp_tiled
from ..optimizer import Optimizer__Union, SoftUpdate
from .reagent_lightning_module import ReAgentLightningModule
from .rl_trainer_pytorch import RLTrainerMixin
from .workspace import NetWorkspace, Pins, backward_wgrad, batch_device, param_grads


class NextSlateValueNormMethod(enum.Enum):
    """How the next slate's summed value is normalised without single selection: by the
    current (NORM_BY_CURRENT_SLATE_SIZE) or the next (NORM_BY_NEXT_SLATE_SIZE) slate size."""
    NORM_BY_CURRENT_SLATE_SIZE = "norm_by_current_slate_size"
    NORM_BY_NEXT_SLATE_SIZE = "norm_by_next_slate_size"


class SlateQTrainer(RLTrainerMixin, ReAgentLightningModule):
    def __init__(self, q_network, q_network_target, slate_size,
                 rl: Optional[RLParameters] = None, optimizer: Optional[Optimizer__Union] = None,
                 slate_opt_parameters: Optional[SlateOptParameters] = None,
                 discount_time_scale: Optional[float] = None, single_selection: bool = True,
                 next_slate_value_norm_method: NextSlateValueNormMethod = (
                     NextSlateValueNormMethod.NORM_BY_CURRENT_SLATE_SIZE),
                 minibatch_size: int = 1024,
                 evaluation: Optional[EvaluationParameters] = None) -> None:
        """rl, optimizer and evaluation default to the reference's field factories:
        RLParameters(maxq_learning=False), Optimizer__Union.default() and
        EvaluationParameters(calc_cpe_in_training=False)."""
        super().__init__()
        self.rl_parameters = RLParameters(maxq_learning=False) if rl is None else rl
        self.discount_time_scale = discount_time_scale
        self.single_selection = single_selection
        # a configuration gives the enum's value as a string
        self.next_slate_value_norm_method = NextSlateValueNormMethod(next_slate_value_norm_method)
        self.q_network = q_network
        self.q_network_target = q_network_target
        self.q_network_optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        self.slate_size = slate_size
        self.slate_opt_parameters = slate_opt_parameters
        self._ws = None
        self._status = None

    def configure_optimizers(self):
        """[Adam(q_network), SoftUpdate] -- :93-110."""
        return [self.q_network_optimizer.make_optimizer_scheduler(self.q_network.parameters()),
                SoftUpdate.make_optimizer_scheduler(list(self.q_network_target.parameters()),
                                                    list(self.q_network.parameters()),
                                                    tau=self.tau)]

    def _check_input(self, batch: rlt.SlateQInput):
        assert isinstance(batch, rlt.SlateQInput), f"learning input is a {type(batch)}"
        assert batch.state.candidate_docs is not None and batch.next_state.candidate_docs is not None
        if self.rl_parameters.maxq_learning:
            # _get_maxq_next_action (:133-143)
            assert self.slate_opt_parameters is not None
            if self.slate_opt_parameters.method != SlateOptMethod.TOP_K:
                raise NotImplementedError(
                    "SlateQ with optimization method other than TOP_K is not implemented.")

    def raise_if_failed(self, wait: bool = True):
        """IndexError if an update met an index outside [-C, C) in action or next_action.
        wait=False only looks at a flag copy that has already reached the host."""
        if self._status is None:
            return
        dev_flag, host_flag, copied = self._status
        if wait:
            copied.synchronize()
        elif not copied.query():
            return
        if int(host_flag[0]) != 0:
            dev_flag.zero_()
            host_flag.zero_()
            raise IndexError("SlateQTrainer: a slate index is outside the candidates [-C, C)")

    # ------------------------------------------------------------------
    def _workspace(self, B, K, C, device):
        key = (B, K, C, device)
        if self._ws is None or self._ws["key"] != key:
            rows = (B + _lib.SLATEQ_ROWS_PER_BLOCK - 1) // _lib.SLATEQ_ROWS_PER_BLOCK
            self._ws = {"key": key,
                        "q": NetWorkspace(self.q_network.arena, B * K, device),
                        "q_cur": torch.empty(B * K, 1, device=device),
                        "q_next": torch.empty(B * C, self.q_network_target.arena.dims[-1],
                                              device=device),
                        "target": torch.empty(B * K, device=device),
                        "mask_count": torch.zeros(1, dtype=torch.int32, device=device),
                        "loss_partials": torch.zeros(rows, device=device),
                        "loss": torch.zeros(1, device=device),
                        "counter": torch.zeros(1, dtype=torch.int32, device=device)}
        if self._status is None or self._status[0].device != device:
            self._status = (torch.zeros(1, dtype=torch.int32, device=device),
                            torch.zeros(1, dtype=torch.int32).pin_memory(), torch.cuda.Event())
        return self._ws

    def _td_step(self, batch: rlt.SlateQInput) -> torch.Tensor:
        self._check_input(batch)
        self.raise_if_failed(wait=False)
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        docs, next_docs = batch.state.candidate_docs, batch.next_state.candidate_docs
        state = pins.tensor(batch.state.float_features)
        B, C, D = docs.float_features.shape
        K = batch.action.shape[1]
        maxq = bool(self.rl_parameters.maxq_learning)
        ws = self._workspace(B, K, C, pins.device)

        # the target network on every next candidate: q_next[b * C + c]
        run_mlp_tiled([self.q_network_target.arena], pins.tensor(batch.next_state.float_features),
                      pins.tensor(next_docs.float_features).view(B * C, D), C, [ws["q_next"]])

        # the taken slate: cat(state.repeat_interleave(K), docs[b, action]).  The gather clamps
        # into [-C, C) so that torch never faults; the head reports what was clamped.
        action = batch.action.to(pins.device, torch.int64).contiguous()
        rows = torch.arange(B, device=pins.device).unsqueeze(1)
        sel = pins.tensor(docs.float_features)[rows, action.clamp(-C, C - 1)]
        x = torch.cat((state.repeat_interleave(K, dim=0), sel.view(B * K, D)), dim=1)
        self._x = x
        self.q_network.arena.forward(x, ws["q_cur"], save=ws["q"])

        a = _lib.SlateqArgsT()
        a.batch, a.num_candidates, a.slate_width = B, C, K
        a.slate_size, a.maxq, a.single_selection = int(self.slate_size), int(maxq), int(self.single_selection)
        a.norm_method = (_lib.SLATEQ_NORM_NEXT if self.next_slate_value_norm_method
                         == NextSlateValueNormMethod.NORM_BY_NEXT_SLATE_SIZE else _lib.SLATEQ_NORM_CURRENT)
        a.q_cur = ws["q_cur"].data_ptr()
        a.q_next = ws["q_next"].data_ptr()
        a.next_value = pins(next_docs.value)
        a.next_mask = pins(next_docs.mask)
        a.cur_mask = pins(docs.mask)
        next_action = None
        if not maxq:
            # _action_docs zeroes the terminal rows of the caller's next_action in place
            next_action = batch.next_action
            if not (next_action.dtype == torch.int64 and next_action.is_contiguous()
                    and next_action.device == pins.device):
                next_action = next_action.to(pins.device, torch.int64).contiguous()
            a.next_width = next_action.shape[1]
            a.next_action = next_action.data_ptr()
        a.action = action.data_ptr()
        a.reward = pins(batch.reward)
        a.reward_mask = pins(batch.reward_mask)
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        if self.discount_time_scale and batch.time_diff is not None:
            td = batch.time_diff.reshape(-1)
            assert td.numel() == B, f"time_diff must hold one value per row, got {tuple(batch.time_diff.shape)}"
            a.time_diff = pins(td)
            a.time_scale = float(self.discount_time_scale)
        a.gamma = float(self.gamma)
        a.dz = ws["q"].dz[-1].data_ptr()
        a.target = ws["target"].data_ptr()
        a.mask_count = ws["mask_count"].data_ptr()
        dev_flag, host_flag, copied = self._status
        a.status = dev_flag.data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        _lib.check(_lib.lib().rb200_slateq_head(a, _lib.cur_stream()), "rb200_slateq_head")
        host_flag.copy_(dev_flag, non_blocking=True)
        copied.record()
        if next_action is not None and next_action is not batch.next_action:
            batch.next_action.copy_(next_action)
        backward_wgrad(self.q_network.arena, ws["q"], x, B * K)
        return ws["loss"].reshape(())

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.SlateQInput, batch_idx: int):
        """Yields the TD loss, then the soft-update result -- :199-276."""
        yield self.fused_loss(self._td_step(training_batch))
        yield self.soft_update_result()

    def train_batch(self, training_batch: rlt.SlateQInput, batch_idx: int = 0,
                    process_group=None):
        self._td_step(training_batch)
        self.adam_step(self.q_network.arena, process_group)
        self.all_batches_processed += 1
        return self._ws["loss"]

    def q_network_grads(self):
        return param_grads(self.q_network.arena, list(self.q_network.parameters()))
