"""QRDQNTrainer with the reference's constructor, optimizer list and generator protocol
(reagent/training/qrdqn_trainer.py:21-227, CPE off).

One update is the distributional step (distributional.py) around rb200_qrdqn_head: mean over
atoms, masked argmax, target distribution, pairwise quantile-Huber loss and d loss / d head
output (:125-155); then rb200_adam_soft_update.  The (N, B, N) pairwise tensor of the
reference (655 MB at config 3) is never materialised.
"""
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import EvaluationParameters, RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .distributional import DistributionalStep
from .dqn_trainer_base import DQNTrainerBaseLightning
from .workspace import check_sample_weight, discount_source


class QRDQNTrainer(DistributionalStep, DQNTrainerBaseLightning):
    def __init__(
        self,
        q_network,
        q_network_target,
        metrics_to_score=None,
        reward_network=None,
        q_network_cpe=None,
        q_network_cpe_target=None,
        actions: Optional[List[str]] = None,
        rl: Optional[RLParameters] = None,
        double_q_learning: bool = True,
        num_atoms: int = 51,
        minibatch_size: int = 1024,
        minibatches_per_step: int = 1,
        optimizer: Optional[Optimizer__Union] = None,
        cpe_optimizer: Optional[Optimizer__Union] = None,
        evaluation: Optional[EvaluationParameters] = None,
    ) -> None:
        rl = RLParameters() if rl is None else rl
        actions = [] if actions is None else actions
        evaluation = EvaluationParameters() if evaluation is None else evaluation
        super().__init__(rl_parameters=rl, metrics_to_score=metrics_to_score, actions=actions,
                         evaluation_parameters=evaluation)
        self.double_q_learning = double_q_learning
        self.minibatch_size = minibatch_size
        self.minibatches_per_step = minibatches_per_step
        self._actions = actions
        self.q_network = q_network
        self.q_network_target = q_network_target
        self.q_network_optimizer = optimizer or Optimizer__Union.default()
        self.num_atoms = num_atoms
        self.register_buffer("quantiles", None)
        self.quantiles = (
            (0.5 + torch.arange(self.num_atoms).float()) / float(self.num_atoms)).view(1, -1)
        self._initialize_cpe(reward_network, q_network_cpe, q_network_cpe_target,
                             optimizer=cpe_optimizer)
        self._ws = None
        self.loss = None

    def configure_optimizers(self):
        optimizers = []
        target_params = list(self.q_network_target.parameters())
        source_params = list(self.q_network.parameters())
        optimizers.append(
            self.q_network_optimizer.make_optimizer_scheduler(self.q_network.parameters()))
        optimizers.append(
            SoftUpdate.make_optimizer_scheduler(target_params, source_params, tau=self.tau))
        return optimizers

    # ------------------------------------------------------------------
    def _launch_head(self, batch, ws, pins, sample_weight):
        B = ws["B"]
        a = _lib.QrdqnArgsT()
        a.batch, a.num_actions, a.num_atoms = B, self.num_actions, self.num_atoms
        a.q_next_online = ws["next_online"].data_ptr()
        a.q_next_target = ws["next_target"].data_ptr()
        a.q_cur = ws["cur"].data_ptr()
        a.action = pins(batch.action)
        a.next_action = pins(batch.next_action)
        a.possible_next_actions_mask = pins(batch.possible_next_actions_mask)
        a.reward = pins(batch.reward.reshape(-1))
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        a.discount_src = pins(discount_source(self, batch))
        a.reward_boost = pins(self.reward_boosts.reshape(-1)) if self._has_reward_boost else None
        a.gamma = float(self.gamma)
        a.double_q = int(bool(self.double_q_learning))
        a.maxq = int(bool(self.maxq_learning))
        a.dz_head = ws["net"].dz[-1].data_ptr()
        a.all_q_values = ws["all_q"].data_ptr()
        a.next_action_idx = ws["next_idx"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        a.sample_weight = pins(check_sample_weight(sample_weight, B))
        _lib.check(_lib.lib().rb200_qrdqn_head(a, _lib.cur_stream()), "rb200_qrdqn_head")

    _qr_step = DistributionalStep._step

    def train_step_gen(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int):
        self._check_input(training_batch)
        loss = self._step(training_batch)
        yield self.fused_loss(loss)
        self.loss = loss.detach()
        if self.has_real_reporter:
            logged_action_idxs = torch.argmax(training_batch.action, dim=1, keepdim=True)
            self.reporter.log(
                td_loss=self.loss, logged_actions=logged_action_idxs,
                logged_rewards=self.boost_rewards(training_batch.reward, training_batch.action),
                model_values=self.all_q_values)
        yield self.soft_update_result()
