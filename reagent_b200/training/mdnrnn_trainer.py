"""MDNRNNTrainer (reagent/training/world_model/mdnrnn_trainer.py): trains a MemoryNetwork to
predict the next state (a gaussian mixture), the reward and non-terminality.  Three launches
per step, then FusedAdam:

  rb200_mdnrnn_forward   LSTM over every step, gmm head, the three losses, dL/d(gmm_outs)
  rb200_mdnrnn_backward  backward through time: dGates of every layer and step
  rb200_mdnrnn_wgrad     weight gradients (split-K partials in the arena's layout)
"""
from typing import Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import MDNRNNTrainerParameters
from ..models.world_model import MdnBuffers, MemoryNetwork, run_forward
from ..optimizer import FusedAdam
from .reagent_lightning_module import ReAgentLightningModule
from .workspace import ensure_gpart, param_grads

LOSS_KEYS = ("gmm", "bce", "mse", "loss")


class MDNRNNTrainer(ReAgentLightningModule):
    """Trainer for MDN-RNN"""

    def __init__(self, memory_network: MemoryNetwork, params: MDNRNNTrainerParameters,
                 cum_loss_hist: int = 100):
        super().__init__()
        if not isinstance(memory_network, MemoryNetwork):
            raise NotImplementedError("MDNRNNTrainer needs a reagent_b200.models.MemoryNetwork "
                                      "(its update runs on the fused kernels); got "
                                      + type(memory_network).__name__)
        self.memory_network = memory_network
        self.params = params
        self._ws: Optional[MdnBuffers] = None

    def configure_optimizers(self):
        """[Adam(mdnrnn, lr)]: torch.optim.Adam(..., foreach=True) with default betas / eps."""
        return [FusedAdam(self.memory_network.mdnrnn.parameters(), lr=self.params.learning_rate)]

    # ------------------------------------------------------------------
    def _step(self, batch: rlt.MemoryNetworkInput, state_dim: Optional[int], train: bool):
        """Forward and losses (and, with `train`, the backward into the gradient partials).
        Returns the device vector [gmm, bce, mse, loss] of the workspace; no host
        synchronisation."""
        assert isinstance(batch, rlt.MemoryNetworkInput)
        net = self.memory_network.mdnrnn
        state = batch.state.float_features
        if state.dim() != 3:
            raise ValueError(f"MDNRNNTrainer: state must be [T, B, state_dim], got "
                             f"{tuple(state.shape)}")
        T, B = state.shape[0], state.shape[1]
        if self._ws is None or not self._ws.fits(T, B, state.device, train):
            self._ws = MdnBuffers(net, T, B, state.device, train)
        ws = self._ws
        p = self.params
        div = 1.0 if state_dim is None else float(state_dim + 2)
        run_forward(net, state, batch.action.float_features, ws,
                    targets=(batch.next_state.float_features, batch.reward, batch.not_terminal),
                    train=train,
                    loss_params=(p.next_state_loss_weight, p.not_terminal_loss_weight,
                                 p.reward_loss_weight, div, int(p.fit_only_one_next_step)))
        if train:
            a = net.args(T, B)
            a.hs, a.cs = ws.hs.data_ptr(), ws.cs.data_ptr()
            a.xin, a.acts, a.dgates, a.dy = (ws.xin.data_ptr(), ws.acts.data_ptr(),
                                             ws.dgates.data_ptr(), ws.dy.data_ptr())
            lib, st = _lib.lib(), _lib.cur_stream()
            _lib.check(lib.rb200_mdnrnn_backward(a, st), "rb200_mdnrnn_backward")
            a.splits = lib.rb200_wgrad_splits(T * B)
            a.gpart = ensure_gpart(net.arena, a.splits).data_ptr()
            _lib.check(lib.rb200_mdnrnn_wgrad(a, st), "rb200_mdnrnn_wgrad")
            net.arena.grad_ready = True
        return ws.loss

    def get_loss(self, training_batch: rlt.MemoryNetworkInput, state_dim: Optional[int] = None):
        """{"gmm", "bce", "mse", "loss"} as device scalars, with
        loss = gmm / (state_dim + 2) + bce + mse when `state_dim` is given, else the sum."""
        losses = self._step(training_batch, state_dim, train=False).clone()
        return dict(zip(LOSS_KEYS, losses.unbind()))

    def _report(self, prefix: str, losses):
        if self.has_real_reporter:
            vals = losses.detach().cpu().tolist()
            self.reporter.log(**{prefix + k: v for k, v in zip(LOSS_KEYS, vals)})

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int):
        """Yields the loss of get_loss(batch, state_dim); its gradients are in the arena."""
        state_dim = training_batch.state.float_features.shape[2]
        losses = self._step(training_batch, state_dim, train=True)
        self._report("", losses)
        loss = losses[3]
        if self.trainer is not None and self.logger is not None:
            self.log("td_loss", loss, prog_bar=True, batch_size=training_batch.batch_size())
        yield self.fused_loss(loss)

    def train_batch(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int = 0):
        """Fast path: the update of train_step_gen plus one FusedAdam launch, with no host
        synchronisation.  Returns the device vector [gmm, bce, mse, loss] (overwritten by
        the next step)."""
        state_dim = training_batch.state.float_features.shape[2]
        losses = self._step(training_batch, state_dim, train=True)
        self.adam_step(self.memory_network.mdnrnn.arena)
        self.all_batches_processed += 1
        return losses

    @torch.no_grad()
    def validation_step(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int):
        state_dim = training_batch.state.float_features.shape[2]
        losses = self.get_loss(training_batch, state_dim)
        self._report("eval_", torch.stack([losses[k] for k in LOSS_KEYS]))
        self.log("td_loss", losses["loss"], prog_bar=True, batch_size=training_batch.batch_size())
        return losses["loss"]

    @torch.no_grad()
    def test_step(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int):
        state_dim = training_batch.state.float_features.shape[2]
        losses = self.get_loss(training_batch, state_dim)
        self._report("test_", torch.stack([losses[k] for k in LOSS_KEYS]))
        self.log("td_loss", losses["loss"], prog_bar=True, batch_size=training_batch.batch_size())
        return losses["loss"]

    def mdnrnn_grads(self):
        """Per-parameter gradients of the last fused backward (inspection / tests)."""
        net = self.memory_network.mdnrnn
        return param_grads(net.arena, list(net.parameters()))
