"""The update QRDQNTrainer and C51Trainer share around their loss heads.  The network
[S -> hidden... -> A*N] runs as a fused trunk + 2-D tiled wide head:

  forward x3             q(s') (double Q only), q_target(s'), q(s) saving its activations
  the trainer's head     rb200_qrdqn_head / rb200_c51_head: targets, loss, d loss / d head output
  rb200_linear_backward_dx (head), rb200_mlp_backward (trunk dZ chain), rb200_mlp_wgrad
"""
from typing import Optional

import torch

from ..core import types as rlt
from .workspace import NetWorkspace, Pins, batch_device, param_grads, wgrad, ws_fits


class DistributionalStep:
    """Mixin of a trainer with q_network / q_network_target of width num_actions * num_atoms and
    a `_launch_head(batch, ws, pins, sample_weight)` that fills and launches its loss head from
    ws["next_online"], ws["next_target"] and ws["cur"] into ws["net"].dz[-1]."""

    def _workspace(self, B, device):
        if not ws_fits(self._ws, B, device):
            arena = self.q_network.arena
            AN = arena.dims[-1]
            self._ws = {
                "B": B, "dev": device,
                "net": NetWorkspace(arena, B, device),
                "next_online": torch.empty(B, AN, device=device),
                "next_target": torch.empty(B, AN, device=device),
                "cur": torch.empty(B, AN, device=device),
                "trunk_tmp": (torch.empty(B, arena.dims[-2], device=device)
                              if len(arena.acts) > 1 else None),
                "all_q": torch.empty(B, self.num_actions, device=device),
                "next_idx": torch.empty(B, dtype=torch.int32, device=device),
                "loss_partials": torch.zeros(B, device=device),
                "loss": torch.zeros(1, device=device),
                "counter": torch.zeros(1, dtype=torch.int32, device=device),
            }
        return self._ws

    def _step(self, batch: rlt.DiscreteDqnInput,
              sample_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Forward, loss head and backward into the gradient partials; returns the device loss
        scalar.  `sample_weight`: [B] fp32 importance weights (loss = mean(w * loss_row), row b of
        the head's dZ scaled by w_b; ws["loss_partials"] keeps the unweighted row losses)."""
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        state = pins.tensor(batch.state.float_features)
        next_state = pins.tensor(batch.next_state.float_features)
        B = state.shape[0]
        ws = self._workspace(B, pins.device)
        qa, ta = self.q_network.arena, self.q_network_target.arena
        net, L = ws["net"], len(qa.acts)
        if qa.dims[-1] != self.num_actions * self.num_atoms:
            raise ValueError("q_network output width must be num_actions * num_atoms")
        qa.refresh()  # no-op for plain MLPs; folds a dueling head into its last Linear
        ta.refresh()
        if self.double_q_learning and self.maxq_learning:
            qa.forward_wide(next_state, ws["next_online"], ws["trunk_tmp"])
        ta.forward_wide(next_state, ws["next_target"], ws["trunk_tmp"])
        qa.forward_wide(state, ws["cur"], net.hidden[L - 2] if L > 1 else None, save=net)
        self._launch_head(batch, ws, pins, sample_weight)
        if L > 1:
            qa.layer_backward_dx(L - 1, net, B, ws)
            if L > 2:
                qa.backward(net, B, n_layers=L - 1)
        wgrad(qa, net, state, B)
        qa.finish_grads()  # dueling: folded-layer gradient -> true parameters
        self.all_q_values = ws["all_q"]
        return ws["loss"].reshape(())

    def train_batch(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int = 0,
                    process_group=None, importance_weights: Optional[torch.Tensor] = None):
        """`importance_weights` ([B] fp32 on the batch's device, prioritized replay): the loss
        becomes mean_b(w_b * loss_b) over the per-row losses and row b of the head gradient is
        scaled by w_b."""
        self._step(training_batch, sample_weight=importance_weights)
        self.adam_step(self.q_network.arena, process_group)
        self.all_batches_processed += 1
        return self._ws["loss"]

    def q_network_grads(self):
        return param_grads(self.q_network.arena, list(self.q_network.parameters()))
