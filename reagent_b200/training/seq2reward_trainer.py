"""Seq2RewardTrainer (reagent/training/world_model/seq2reward_trainer.py): trains a
Seq2RewardNetwork to predict the discounted reward accumulated up to each sequence's last valid
step, and a step-prediction MLP to predict that step.  Per update:

  rb200_seq2reward_forward   LSTM, acc_reward, target, MSE, dL/dacc_reward, step labels
  rb200_seq2reward_backward  backward through time, dh0
  rb200_seq2reward_wgrad     weight gradients (split-K partials in the arena's layout)
  rb200_mlp_forward, rb200_bc_xent_head, rb200_mlp_backward, rb200_mlp_wgrad   step network

then one FusedAdam launch per network.  get_Q runs the prefix-tree plan (rb200_seq2reward_plan).
"""
import logging
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib
from ..core import types as rlt
from ..core.parameters import Seq2RewardTrainerParameters
from ..models.fully_connected_network import FullyConnectedNetwork
from ..models.seq2reward_model import (Seq2RewardBuffers, Seq2RewardNetwork, backward_wgrad,
                                       run_forward)
from ..optimizer import FusedAdam
from .reagent_lightning_module import ReAgentLightningModule
from .workspace import NetWorkspace, ensure_gpart, param_grads
from .workspace import backward_wgrad as mlp_backward_wgrad

logger = logging.getLogger(__name__)


def gen_permutations(seq_len: int, num_action: int) -> torch.Tensor:
    """All seq_len action sequences in lexical order, one-hot: [seq_len, num_action ** seq_len,
    num_action] (reagent/training/utils.py)."""
    all_permut = torch.cartesian_prod(*[torch.arange(num_action)] * seq_len)
    if seq_len == 1:
        all_permut = all_permut.unsqueeze(1)
    all_permut = F.one_hot(all_permut, num_action).transpose(0, 1)
    return all_permut.float()


def _check_permutations(all_permut: torch.Tensor):
    """(k, A) of `all_permut`, which must be gen_permutations(k, A): the plan enumerates the
    sequences itself.  Checked once per tensor."""
    if all_permut.dim() != 3:
        raise ValueError(f"get_Q: all_permut must be [seq_len, num_perm, num_action], got "
                         f"{tuple(all_permut.shape)}")
    k, _, A = all_permut.shape
    if getattr(all_permut, "_rb200_checked_version", None) != all_permut._version:
        if not torch.equal(all_permut.detach().float().cpu(), gen_permutations(k, A)):
            raise ValueError("get_Q: all_permut is not gen_permutations(seq_len, num_action); "
                             "the fused plan enumerates every sequence in lexical order")
        all_permut._rb200_checked_version = all_permut._version
    return k, A


@torch.no_grad()
def get_step_prediction(step_predict_network: FullyConnectedNetwork,
                        training_batch: rlt.MemoryNetworkInput):
    first_step_state = training_batch.state.float_features[0]
    pred_step = step_predict_network(first_step_state)
    return F.softmax(pred_step, dim=1)


@torch.no_grad()
def get_Q(seq2reward_network: Seq2RewardNetwork, cur_state: torch.Tensor,
          all_permut: torch.Tensor) -> torch.Tensor:
    """[B, A]: for each first action, the max predicted accumulated reward over the sequences
    of all_permut ([seq_len, A ** seq_len, A], gen_permutations) that start with it."""
    k, A = _check_permutations(all_permut)
    if A != seq2reward_network.action_dim:
        raise ValueError(f"get_Q: all_permut has {A} actions, the network {seq2reward_network.action_dim}")
    return seq2reward_network.plan(cur_state, k)[0]


@torch.no_grad()
def plan_short_sequence_q(seq2reward_network: Seq2RewardNetwork,
                          step_predict_network: FullyConnectedNetwork, state: torch.Tensor,
                          seq_len: int, num_action: int) -> torch.Tensor:
    """[B, A]: sum_s softmax(step_predict_network(state))[:, s] * Q_{s+1}(state), the planning
    of Seq2RewardPlanShortSeqWithPreprocessor.forward without the preprocessor.  Every horizon
    comes from one prefix-tree plan; the weighting over [B, seq_len, A] runs in torch."""
    if num_action != seq2reward_network.action_dim:
        raise ValueError(f"plan_short_sequence_q: num_action {num_action} != the network's "
                         f"{seq2reward_network.action_dim}")
    step_probability = F.softmax(step_predict_network(state), dim=1)
    _, q_all = seq2reward_network.plan(state, seq_len, all_horizons=True)
    return torch.sum(q_all * step_probability.unsqueeze(2), dim=1)


class Seq2RewardTrainer(ReAgentLightningModule):
    """Trainer for Seq2Reward"""

    def __init__(self, seq2reward_network: Seq2RewardNetwork,
                 params: Seq2RewardTrainerParameters):
        super().__init__()
        if not isinstance(seq2reward_network, Seq2RewardNetwork):
            raise NotImplementedError("Seq2RewardTrainer needs a reagent_b200.models."
                                      "Seq2RewardNetwork (its update runs on the fused kernels); "
                                      "got " + type(seq2reward_network).__name__)
        self.seq2reward_network = seq2reward_network
        self.params = params
        # Turning off Q value output during training:
        self.view_q_value = params.view_q_value
        # permutations used to do planning
        self.all_permut = gen_permutations(params.multi_steps, len(self.params.action_names))
        self.mse_loss = nn.MSELoss(reduction="mean")
        # Predict how many steps are remaining from the current step
        self.step_predict_network = FullyConnectedNetwork(
            [self.seq2reward_network.state_dim, self.params.step_predict_net_size,
             self.params.step_predict_net_size, self.params.multi_steps],
            ["relu", "relu", "linear"], use_layer_norm=False)
        self.step_loss = nn.CrossEntropyLoss(reduction="mean")
        self._ws: Optional[Seq2RewardBuffers] = None
        self._step_ws = None

    def configure_optimizers(self):
        """[Adam(seq2reward_network), Adam(step_predict_network)], both at learning_rate:
        torch.optim.Adam(..., foreach=True) with default betas / eps."""
        return [FusedAdam(self.seq2reward_network.parameters(), lr=self.params.learning_rate),
                FusedAdam(self.step_predict_network.parameters(), lr=self.params.learning_rate)]

    # ------------------------------------------------------------------
    def _check_valid_step(self, batch: rlt.MemoryNetworkInput):
        """1 <= valid_step <= min(seq_len, multi_steps), as the reference's indexing and cross
        entropy need (host synchronisation)."""
        if batch.valid_step is None:
            raise ValueError("Seq2RewardTrainer: the batch has no valid_step")
        T = batch.action.float_features.shape[0]
        hi = min(T, self.params.multi_steps)
        v = batch.valid_step.flatten()
        if v.numel() and (int(v.min()) < 1 or int(v.max()) > hi):
            raise ValueError(f"Seq2RewardTrainer: valid_step must lie in [1, {hi}] "
                             f"(min(seq_len, multi_steps)), got [{int(v.min())}, {int(v.max())}]")

    def _step(self, batch: rlt.MemoryNetworkInput, train: bool):
        """Both losses (and with `train` both backwards into the gradient partials).  Returns
        the device scalars (mse, step cross entropy); no host synchronisation."""
        assert isinstance(batch, rlt.MemoryNetworkInput)
        if batch.valid_step is None:
            raise ValueError("Seq2RewardTrainer: the batch has no valid_step (the target and the "
                             "step labels are read at valid_step - 1)")
        net = self.seq2reward_network
        state, action = batch.state.float_features, batch.action.float_features
        if state.dim() != 3 or action.dim() != 3:
            raise ValueError(f"Seq2RewardTrainer: state and action must be [T, B, dim], got "
                             f"{tuple(state.shape)} and {tuple(action.shape)}")
        if not state.is_cuda:
            raise _lib.Rb200Error("Seq2RewardTrainer: training batch must be on the GPU "
                                  "(reagent_b200 has no CPU path)")
        T, B, k = action.shape[0], action.shape[1], self.params.multi_steps
        if self._ws is None or not self._ws.fits(T, B, k, state.device, train):
            self._ws = Seq2RewardBuffers(net, T, B, k, state.device, train)
        ws = self._ws
        run_forward(net, state, action, batch.valid_step.flatten(), ws, reward=batch.reward,
                    gamma=self.params.gamma, train=train, multi_steps=k)
        if train:
            splits = _lib.lib().rb200_wgrad_splits(T * B)
            backward_wgrad(net, ws, splits, ensure_gpart(net.arena, splits))
        # the step network: cross entropy against the one-hot labels of valid_step - 1
        ar = self.step_predict_network.arena
        state0 = ws.keep[0]
        sw = self._step_ws
        if sw is None or sw["B"] != B or sw["dev"] != state.device:
            sw = self._step_ws = {
                "B": B, "dev": state.device, "net": NetWorkspace(ar, B, state.device),
                "scores": torch.empty(B, k, device=state.device),
                "mask": torch.ones(B, k, device=state.device),
                "loss_partials": torch.zeros(-(-B // _lib.BC_ROWS_PER_BLOCK), device=state.device),
                "loss": torch.zeros(1, device=state.device),
                "counter": torch.zeros(1, dtype=torch.int32, device=state.device)}
        ar.forward(state0, sw["scores"], save=sw["net"] if train else None)
        a = _lib.BcXentArgsT()
        a.batch, a.num_actions = B, k
        a.logits, a.labels, a.mask = (sw["scores"].data_ptr(), ws.step_labels.data_ptr(),
                                      sw["mask"].data_ptr())
        a.dz = sw["net"].dz[-1].data_ptr() if train else None
        a.loss_partials, a.loss = sw["loss_partials"].data_ptr(), sw["loss"].data_ptr()
        a.tile_counter = sw["counter"].data_ptr()
        _lib.check(_lib.lib().rb200_bc_xent_head(a, _lib.cur_stream()), "rb200_bc_xent_head")
        if train:
            mlp_backward_wgrad(ar, sw["net"], state0, B)
        return ws.loss.reshape(()), sw["loss"].reshape(())

    def get_mse_loss(self, training_batch: rlt.MemoryNetworkInput):
        return self._step(training_batch, train=False)[0].clone()

    def get_step_entropy_loss(self, training_batch: rlt.MemoryNetworkInput):
        return self._step(training_batch, train=False)[1].clone()

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int):
        """Yields the MSE, then the step cross entropy; their gradients are in the arenas."""
        self._check_valid_step(training_batch)
        mse_loss, step_entropy_loss = self._step(training_batch, train=True)
        yield self.fused_loss(mse_loss)
        if self.view_q_value or self.has_real_reporter:
            detached_mse_loss = mse_loss.item()
            detached_step_entropy_loss = step_entropy_loss.item()
            if self.view_q_value:
                state_first_step = training_batch.state.float_features[0]
                q_values = get_Q(self.seq2reward_network, state_first_step,
                                 self.all_permut).cpu().mean(0).tolist()
            else:
                q_values = [0] * len(self.params.action_names)
            step_probability = get_step_prediction(
                self.step_predict_network, training_batch).cpu().mean(dim=0).numpy()
            logger.info(f"Seq2Reward trainer output: mse_loss={detached_mse_loss}, "
                        f"step_entropy_loss={detached_step_entropy_loss}, q_values={q_values}, "
                        f"step_probability={step_probability}")
            if self.has_real_reporter:
                self.reporter.log(mse_loss=detached_mse_loss,
                                  step_entropy_loss=detached_step_entropy_loss,
                                  q_values=[q_values])
        yield self.fused_loss(step_entropy_loss)

    def train_batch(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int = 0):
        """Fast path: the update of train_step_gen plus one FusedAdam launch per network, with
        no host synchronisation and no valid_step check.  Returns the device scalars (mse,
        step cross entropy), overwritten by the next step."""
        losses = self._step(training_batch, train=True)
        self.adam_step(self.seq2reward_network.arena)
        self.adam_step(self.step_predict_network.arena)
        self.all_batches_processed += 1
        return losses

    @torch.no_grad()
    def validation_step(self, batch: rlt.MemoryNetworkInput, batch_idx: int):
        self._check_valid_step(batch)
        mse, step = self._step(batch, train=False)
        detached_mse_loss = mse.item()
        detached_step_entropy_loss = step.item()
        state_first_step = batch.state.float_features[0]
        # shape: batch_size, action_dim
        q_values_all_action_all_data = get_Q(self.seq2reward_network, state_first_step,
                                             self.all_permut).cpu()
        q_values = q_values_all_action_all_data.mean(0).tolist()
        action_distribution = torch.bincount(torch.argmax(q_values_all_action_all_data, dim=1),
                                             minlength=len(self.params.action_names))
        action_distribution = (action_distribution.float()
                               / torch.sum(action_distribution)).tolist()
        if self.has_real_reporter:
            self.reporter.log(eval_mse_loss=detached_mse_loss,
                              eval_step_entropy_loss=detached_step_entropy_loss,
                              eval_q_values=[q_values],
                              eval_action_distribution=[action_distribution])
        return (detached_mse_loss, detached_step_entropy_loss, q_values, action_distribution)

    def warm_start_components(self):
        return ["seq2reward_network"]

    def seq2reward_grads(self):
        """Per-parameter gradients of the last fused backward (inspection / tests)."""
        net = self.seq2reward_network
        return param_grads(net.arena, list(net.parameters()))

    def step_predict_grads(self):
        net = self.step_predict_network
        return param_grads(net.arena, list(net.parameters()))
