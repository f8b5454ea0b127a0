"""C51Trainer (reagent/training/c51_trainer.py:20-214): categorical distributional DQN.  The
distributional network (trunk + wide [hidden -> A*N] head) runs on the step it shares with
QR-DQN (distributional.py); rb200_c51_head does the log-softmax, masked arg max, categorical
projection, cross-entropy loss and d loss / d logits, one CTA per batch row."""
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .distributional import DistributionalStep
from .reagent_lightning_module import ReAgentLightningModule
from .rl_trainer_pytorch import RLTrainerMixin
from .workspace import check_sample_weight, discount_source, register_reward_boosts


class C51Trainer(DistributionalStep, RLTrainerMixin, ReAgentLightningModule):
    def __init__(self, q_network, q_network_target, actions: Optional[List[str]] = None,
                 rl: Optional[RLParameters] = None, double_q_learning: bool = True,
                 minibatch_size: int = 1024, minibatches_per_step: int = 1, num_atoms: int = 51,
                 qmin: float = -100, qmax: float = 200,
                 optimizer: Optional[Optimizer__Union] = None) -> None:
        super().__init__()
        self.double_q_learning = double_q_learning
        self.minibatch_size = minibatch_size
        self.minibatches_per_step = minibatches_per_step
        self._actions = [] if actions is None else actions
        self.q_network = q_network
        self.q_network_target = q_network_target
        self.q_network_optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        self.qmin, self.qmax, self.num_atoms = qmin, qmax, num_atoms
        self.rl_parameters = RLParameters() if rl is None else rl
        self.register_buffer("support", torch.linspace(self.qmin, self.qmax, self.num_atoms))
        self.scale_support = (self.qmax - self.qmin) / (self.num_atoms - 1.0)
        register_reward_boosts(self, self._actions, self.rl_parameters.reward_boost)
        self._ws = None

    @property
    def num_actions(self) -> int:
        return len(self._actions)

    def configure_optimizers(self):
        return [self.q_network_optimizer.make_optimizer_scheduler(self.q_network.parameters()),
                SoftUpdate.make_optimizer_scheduler(list(self.q_network_target.parameters()),
                                                    list(self.q_network.parameters()), tau=self.tau)]

    def _launch_head(self, batch, ws, pins, sample_weight):
        B = ws["B"]
        dq = self.double_q_learning and self.maxq_learning
        a = _lib.C51ArgsT()
        a.batch, a.num_actions, a.num_atoms = B, self.num_actions, self.num_atoms
        a.logits_next_online = ws["next_online"].data_ptr() if dq else None
        a.logits_next_target = ws["next_target"].data_ptr()
        a.logits_cur = ws["cur"].data_ptr()
        a.action = pins(batch.action)
        a.next_action = pins(batch.next_action)
        a.possible_next_actions_mask = pins(batch.possible_next_actions_mask)
        a.reward = pins(batch.reward.reshape(-1))
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        a.discount_src = pins(discount_source(self, batch))
        a.reward_boost = pins(self.reward_boosts.reshape(-1)) if self._has_reward_boost else None
        a.support = pins(self.support)
        a.gamma, a.qmin, a.qmax = float(self.gamma), float(self.qmin), float(self.qmax)
        a.scale_support = float(self.scale_support)
        a.double_q, a.maxq = int(bool(self.double_q_learning)), int(bool(self.maxq_learning))
        a.dz_logits = ws["net"].dz[-1].data_ptr()
        a.all_q_values = ws["all_q"].data_ptr()
        a.next_action_idx = ws["next_idx"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        a.sample_weight = pins(check_sample_weight(sample_weight, B))
        _lib.check(_lib.lib().rb200_c51_head(a, _lib.cur_stream()), "rb200_c51_head")

    _c51_step = DistributionalStep._step

    def train_step_gen(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int):
        loss = self._step(training_batch)
        yield self.fused_loss(loss)
        yield self.soft_update_result()

    @torch.no_grad()
    def boost_rewards(self, rewards: torch.Tensor, actions: torch.Tensor) -> torch.Tensor:
        return rewards + torch.sum(actions.float() * self.reward_boosts, dim=1, keepdim=True)

    def argmax_with_mask(self, q_values, possible_actions_mask):
        q_values = q_values.reshape(possible_actions_mask.shape)
        return (q_values + (-1e9) * (1 - possible_actions_mask)).argmax(1)
