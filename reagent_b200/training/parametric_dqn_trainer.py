"""ParametricDQNTrainer (reagent/training/parametric_dqn_trainer.py:22-214) on the generic
kernels of this library: the critic-shaped q_network(state, action) is evaluated by
rb200_mlp_forward, and for max-Q learning by rb200_mlp_forward_tiled, which scores every
(next state, possible next action) pair of both networks in one launch without writing the
tiled input to HBM.  rb200_pdqn_head turns the values into the TD loss and d loss / d q,
rb200_mlp_backward + rb200_mlp_wgrad produce the parameter gradients, FusedAdam / SoftUpdate
apply them.  The concatenation of (state, action) for the current-state and SARSA forwards is
torch plumbing on device tensors."""
from typing import Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import RLParameters
from ..models.arena import run_mlp_tiled
from ..optimizer import Optimizer__Union, SoftUpdate
from .reagent_lightning_module import ReAgentLightningModule
from .rl_trainer_pytorch import RLTrainerMixin
from .workspace import (NetWorkspace, Pins, backward_wgrad, batch_device, discount_source,
                        loss_kind, param_grads, ws_fits)


class ParametricDQNTrainer(RLTrainerMixin, ReAgentLightningModule):
    def __init__(self, q_network, q_network_target, reward_network=None,
                 rl: Optional[RLParameters] = None, double_q_learning: bool = True,
                 minibatches_per_step: int = 1, optimizer: Optional[Optimizer__Union] = None,
                 log_tensorboard: bool = False) -> None:
        super().__init__()
        self.rl_parameters = RLParameters() if rl is None else rl
        self.double_q_learning = double_q_learning
        self.minibatches_per_step = minibatches_per_step or 1
        self.q_network = q_network
        self.q_network_target = q_network_target
        self.reward_network = reward_network
        self.optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        self.log_tensorboard = log_tensorboard
        if self.rl_parameters.q_network_loss == "bce_with_logits":
            raise NotImplementedError("bce_with_logits (gamma == 0 only) has no fused head")
        self.q_network_loss_kind = loss_kind(self.rl_parameters.q_network_loss)
        self._ws = None

    @property
    def num_actions(self) -> int:
        """Width of the q network's action input: the one-hot width of replay batches
        (ReplayBuffer.sample_parametric_dqn_batch) and of the act-time policy."""
        return self.q_network.action_dim

    def configure_optimizers(self):
        """[Adam(q_network), (Adam(reward_network),) SoftUpdate] -- :66-86."""
        optimizers = [self.optimizer.make_optimizer_scheduler(self.q_network.parameters())]
        if self.reward_network is not None:
            optimizers.append(self.optimizer.make_optimizer_scheduler(self.reward_network.parameters()))
        optimizers.append(SoftUpdate.make_optimizer_scheduler(
            list(self.q_network_target.parameters()), list(self.q_network.parameters()), tau=self.tau))
        return optimizers

    def _check_input(self, training_batch: rlt.ParametricDqnInput):
        assert isinstance(training_batch, rlt.ParametricDqnInput)
        assert training_batch.not_terminal.dim() == training_batch.reward.dim() == 2
        assert training_batch.not_terminal.shape[1] == training_batch.reward.shape[1] == 1
        assert (training_batch.action.float_features.dim()
                == training_batch.next_action.float_features.dim() == 2)

    # ------------------------------------------------------------------
    def _workspace(self, B, device):
        if not ws_fits(self._ws, B, device):
            self._ws = {"B": B, "dev": device,
                        "q": NetWorkspace(self.q_network.arena, B, device),
                        "r": (None if self.reward_network is None
                              else NetWorkspace(self.reward_network.arena, B, device)),
                        "q_values": torch.empty(B, 1, device=device),
                        "td_target": torch.empty(B, device=device),
                        "loss_partials": torch.zeros((B + 255) // 256, device=device),
                        "loss": torch.zeros(1, device=device),
                        "r_loss": torch.zeros(1, device=device),
                        "counter": torch.zeros(1, dtype=torch.int32, device=device)}
        return self._ws

    @staticmethod
    def _fwd(net, x):
        out = torch.empty(x.shape[0], net.arena.dims[-1], device=x.device)
        net.arena.forward(x, out)
        return out

    def _td_step(self, batch: rlt.ParametricDqnInput) -> torch.Tensor:
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        state = batch.state.float_features.float().contiguous()
        B = state.shape[0]
        ws = self._workspace(B, pins.device)
        a = _lib.PdqnArgsT()
        a.batch = B
        next_state = batch.next_state.float_features.float()
        if self.maxq_learning:
            pna = pins.tensor(batch.possible_next_actions.float_features)
            product = pna.shape[0]
            assert product % B == 0, f"batch_size * max_num_action {product} is not divisible by batch_size {B}"
            M = product // B
            # FeatureData.get_tiled_batch + cat with the possible next actions, built per row
            # tile in shared memory; both networks score the same tile in one launch
            ns = pins.tensor(next_state)
            nq_t = torch.empty(product, self.q_network_target.arena.dims[-1], device=pins.device)
            arenas, outs = [self.q_network_target.arena], [nq_t]
            nq = None
            if self.double_q_learning:
                nq = torch.empty_like(nq_t)
                arenas.append(self.q_network.arena)
                outs.append(nq)
            run_mlp_tiled(arenas, ns, pna, M, outs)
            pins.keep += [nq_t, nq]
            a.max_num_action = M
            a.next_q = None if nq is None else nq.data_ptr()
            a.next_q_target = nq_t.data_ptr()
            a.mask = pins(batch.possible_next_actions_mask)
        else:  # SARSA on the target network
            x_next = torch.cat((next_state, batch.next_action.float_features.float()), dim=1).contiguous()
            nq_t = self._fwd(self.q_network_target, x_next)
            pins.keep += [x_next, nq_t]
            a.max_num_action = 0
            a.next_q_target = nq_t.data_ptr()
        a.reward = pins(batch.reward.reshape(-1))
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        a.gamma = float(self.gamma)
        src = discount_source(self, batch)
        a.discount_src = pins(src)
        a.discount_mode = _lib.DISCOUNT_CONST if src is None else _lib.DISCOUNT_POW
        a.double_q = int(bool(self.double_q_learning))
        a.loss_kind = self.q_network_loss_kind
        x = torch.cat((state, batch.action.float_features.float()), dim=1).contiguous()
        self._x = x
        qv = ws["q_values"]
        self.q_network.arena.forward(x, qv, save=ws["q"])
        a.q_values = qv.data_ptr()
        a.dz = ws["q"].dz[-1].data_ptr()
        a.td_target = ws["td_target"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        _lib.check(_lib.lib().rb200_pdqn_head(a, _lib.cur_stream()), "rb200_pdqn_head")
        backward_wgrad(self.q_network.arena, ws["q"], x, B)
        return ws["loss"].reshape(())

    def _reward_step(self, batch: rlt.ParametricDqnInput) -> torch.Tensor:
        """mse(reward_network(state, action), cat(reward, metrics)) -- :176-190."""
        ws = self._ws
        x, B = self._x, self._x.shape[0]
        metrics = batch.extras.metrics if batch.extras is not None else None
        mrc = batch.reward if metrics is None else torch.cat((batch.reward, metrics), dim=1)
        w = ws["r"]
        est = torch.empty(B, self.reward_network.arena.dims[-1], device=x.device)
        self.reward_network.arena.forward(x, est, save=w)
        diff = est - mrc.float()
        w.dz[-1].copy_(diff * (2.0 / diff.numel()))
        ws["r_loss"].copy_((diff * diff).mean().reshape(1))
        backward_wgrad(self.reward_network.arena, w, x, B)
        return ws["r_loss"].reshape(())

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.ParametricDqnInput, batch_idx: int):
        self._check_input(training_batch)
        td_loss = self._td_step(training_batch)
        yield self.fused_loss(td_loss)
        if self.reward_network is not None:
            yield self.fused_loss(self._reward_step(training_batch))
        yield self.soft_update_result()

    def train_batch(self, training_batch: rlt.ParametricDqnInput, batch_idx: int = 0,
                    process_group=None):
        self._td_step(training_batch)
        self.adam_step(self.q_network.arena, process_group)
        if self.reward_network is not None:
            self._reward_step(training_batch)
            self.adam_step(self.reward_network.arena, process_group)
        self.all_batches_processed += 1
        return self._ws["loss"]

    def q_network_grads(self):
        return param_grads(self.q_network.arena, list(self.q_network.parameters()))
