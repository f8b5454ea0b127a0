"""BehavioralCloningTrainer (reagent/training/behavioral_cloning_trainer.py:17-83): a supervised
update of a FullyConnectedDQN towards the logged actions, e.g. to train the imitator of
DQNTrainer(imitator=..., bcq=BCQConfig(...)).  Four launches per step:

  rb200_mlp_forward     scores, saving the activations            bc_net(state)
  rb200_bc_xent_head    masked logits, mean cross entropy, dL/dz   :38-56, models/dqn.py:55-63
  rb200_mlp_backward    dZ chain of the hidden layers              autograd
  rb200_mlp_wgrad       weight gradients (split-K partials)        autograd Linear backward

then FusedAdam.  The label of a row is the arg max of its own one-hot action (dim 1); see
DESIGN.md section 4 for how that relates to the reference's `labels.max(dim=0)`.
"""
from typing import Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..optimizer import Optimizer__Union
from .reagent_lightning_module import ReAgentLightningModule
from .workspace import NetWorkspace, Pins, backward_wgrad, batch_device, param_grads, ws_fits


class BehavioralCloningTrainer(ReAgentLightningModule):
    def __init__(self, bc_net, optimizer: Optional[Optimizer__Union] = None) -> None:
        from ..models.dqn import FullyConnectedDQN

        super().__init__()
        if not isinstance(bc_net, FullyConnectedDQN) or bc_net.num_atoms is not None:
            raise NotImplementedError(
                "BehavioralCloningTrainer needs a reagent_b200.models.FullyConnectedDQN without "
                "atoms (its forward runs on the fused MLP kernel); got " + type(bc_net).__name__)
        self.bc_net = bc_net
        # field(default_factory=Optimizer__Union.default) in the reference
        self.optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        self._ws = None

    def configure_optimizers(self):
        """[Adam(bc_net)] -- :30-35."""
        return [self.optimizer.make_optimizer_scheduler(self.bc_net.parameters())]

    # ------------------------------------------------------------------
    def _workspace(self, B: int, device):
        if not ws_fits(self._ws, B, device):
            self._ws = {"B": B, "dev": device,
                        "net": NetWorkspace(self.bc_net.arena, B, device),
                        "scores": torch.empty(B, self.bc_net.action_dim, device=device),
                        "loss_partials": torch.zeros(-(-B // _lib.BC_ROWS_PER_BLOCK),
                                                     device=device),
                        "loss": torch.zeros(1, device=device),
                        "counter": torch.zeros(1, dtype=torch.int32, device=device)}
        return self._ws

    def _step(self, batch: rlt.BehavioralCloningModelInput, do_backward: bool = True) -> torch.Tensor:
        """Forward, loss head (and backward into the gradient partials).  Returns the device
        loss scalar (shape []); no host synchronisation."""
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        state = pins.tensor(batch.state.float_features)
        ar = self.bc_net.arena
        B, A = state.shape[0], self.bc_net.action_dim
        if state.shape[1] != ar.dims[0]:
            raise ValueError(f"state has {state.shape[1]} features, bc_net expects {ar.dims[0]}")
        if batch.possible_actions_mask is None:
            raise TypeError("BehavioralCloningTrainer needs possible_actions_mask")
        labels = pins.tensor(batch.action)
        mask = pins.tensor(batch.possible_actions_mask)
        for name, t in (("action", labels), ("possible_actions_mask", mask)):
            if tuple(t.shape) != (B, A):
                raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {(B, A)}")
        ws = self._workspace(B, pins.device)
        net = ws["net"]
        ar.forward(state, ws["scores"], save=net if do_backward else None)
        a = self._xent_args(ws, labels, mask, do_backward)
        _lib.check(_lib.lib().rb200_bc_xent_head(a, _lib.cur_stream()), "rb200_bc_xent_head")
        if do_backward:
            backward_wgrad(ar, net, state, B)
        return ws["loss"].reshape(())

    def _xent_args(self, ws, labels: torch.Tensor, mask: torch.Tensor, do_backward: bool = True):
        """The loss head's arguments on workspace `ws`, for the fp32 [B, A] device tensors
        `labels` (one-hot) and `mask`."""
        a = _lib.BcXentArgsT()
        a.batch, a.num_actions = ws["B"], self.bc_net.action_dim
        a.logits, a.labels, a.mask = ws["scores"].data_ptr(), labels.data_ptr(), mask.data_ptr()
        a.dz = ws["net"].dz[-1].data_ptr() if do_backward else None
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        return a

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.BehavioralCloningModelInput, batch_idx: int):
        """Yields the cross-entropy loss -- :43-56."""
        self._check_input(training_batch)
        loss = self._step(training_batch)
        if self.has_real_reporter:
            self.reporter.log(loss=loss.detach().cpu())
        yield self.fused_loss(loss)

    def train_batch(self, training_batch: rlt.BehavioralCloningModelInput, batch_idx: int = 0,
                    process_group=None):
        """Fast path: the update of train_step_gen + one FusedAdam launch, with no host
        synchronisation and without the data checks of _check_input.  With `process_group`
        (data parallel, equal shards per rank) the gradient is averaged over the ranks before
        Adam, as in DQNTrainer.train_batch."""
        self._step(training_batch)
        self.adam_step(self.bc_net.arena, process_group)
        self.all_batches_processed += 1
        return self._ws["loss"]

    @torch.no_grad()
    def validation_step(self, batch: rlt.BehavioralCloningModelInput, batch_idx: int):
        """The detached CPU loss of the same computation, without gradients -- :59-68."""
        self._check_input(batch)
        return self._step(batch, do_backward=False).detach().cpu()

    def bc_net_grads(self):
        """Per-parameter gradients of the last fused backward (inspection / tests)."""
        return param_grads(self.bc_net.arena, list(self.bc_net.parameters()))

    def _check_input(self, training_batch: rlt.BehavioralCloningModelInput):
        """:70-83: one-hot labels with more than one row, none of them masked out."""
        assert isinstance(training_batch, rlt.BehavioralCloningModelInput)
        labels = training_batch.action
        if not (len(labels.shape) > 1 and labels.shape[0] > 1):
            raise TypeError("label tensor format or dimension does not match loss function")
        mask = training_batch.possible_actions_mask
        if mask is None:
            raise TypeError("BehavioralCloningTrainer needs possible_actions_mask (the reference "
                            "multiplies the labels by it)")
        assert torch.all(labels * mask == labels)  # check all labels are not masked out
