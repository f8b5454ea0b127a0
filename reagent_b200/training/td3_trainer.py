"""TD3Trainer with the reference's constructor, optimizer order and generator protocol
(reagent/training/td3_trainer.py:20-199).

  rb200_ac_critic_step  target actor + clipped noise, min of target critics, q1/q2 losses
                        and critic dZ chains                          td3_trainer.py:138-178
  wgrad x2, Adam(q1), Adam(q2)
  every `delayed_policy_update`-th batch:
  rb200_ac_actor_step   -mean(q1(s, actor(s))) and its backward through q1   :181-187
  wgrad, Adam(actor), SoftUpdate(q1, q2, actor targets)                       :189-194
  otherwise the 3rd and 4th yields are None (:196-199).
`noise_variance` multiplies the N(0,1) draw (it acts as a std-dev, :141).
"""
import copy
from typing import Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .actor_critic_base import ActorCriticBase


class TD3Trainer(ActorCriticBase):
    ALGO = _lib.ALGO_TD3

    def __init__(
        self,
        actor_network,
        q1_network,
        q2_network=None,
        rl: Optional[RLParameters] = None,
        q_network_optimizer: Optional[Optimizer__Union] = None,
        actor_network_optimizer: Optional[Optimizer__Union] = None,
        minibatch_size: int = 64,
        noise_variance: float = 0.2,
        noise_clip: float = 0.5,
        delayed_policy_update: int = 2,
        minibatches_per_step: int = 1,
    ) -> None:
        super().__init__()
        self._ac_init()
        self.rl_parameters = RLParameters() if rl is None else rl
        self.minibatch_size = minibatch_size
        self.minibatches_per_step = minibatches_per_step or 1
        self.q1_network = q1_network
        self.q1_network_target = copy.deepcopy(self.q1_network)
        self.q_network_optimizer = q_network_optimizer or Optimizer__Union.default()
        self.q2_network = q2_network
        if self.q2_network is not None:
            self.q2_network_target = copy.deepcopy(self.q2_network)
        else:
            self.q2_network_target = None
        self.actor_network = actor_network
        self.actor_network_target = copy.deepcopy(self.actor_network)
        self.actor_network_optimizer = actor_network_optimizer or Optimizer__Union.default()
        self.noise_variance = noise_variance
        self.noise_clip_range = (-noise_clip, noise_clip)
        self.delayed_policy_update = delayed_policy_update

    def configure_optimizers(self):
        """q1, q2, actor, SoftUpdate(q1, q2, actor) (td3_trainer.py:89-123)."""
        optimizers = []
        optimizers.append(
            self.q_network_optimizer.make_optimizer_scheduler(self.q1_network.parameters()))
        if self.q2_network:
            optimizers.append(
                self.q_network_optimizer.make_optimizer_scheduler(self.q2_network.parameters()))
        optimizers.append(
            self.actor_network_optimizer.make_optimizer_scheduler(
                self.actor_network.parameters()))
        target_params = list(self.q1_network_target.parameters())
        source_params = list(self.q1_network.parameters())
        if self.q2_network:
            target_params += list(self.q2_network_target.parameters())
            source_params += list(self.q2_network.parameters())
        target_params += list(self.actor_network_target.parameters())
        source_params += list(self.actor_network.parameters())
        optimizers.append(
            SoftUpdate.make_optimizer_scheduler(target_params, source_params, tau=self.tau))
        return optimizers

    def _fill(self, a, pins):
        a.noise_variance = float(self.noise_variance)
        a.noise_clip = float(self.noise_clip_range[1])

    def train_step_gen(self, training_batch: rlt.PolicyNetworkInput, batch_idx: int):
        assert isinstance(training_batch, rlt.PolicyNetworkInput)
        closs = self._critic_step(training_batch, self.actor_network_target,
                                  self.q1_network_target, self.q2_network_target, self._fill)
        self.log("td_loss", closs[0], prog_bar=True)
        yield self.fused_loss(closs[0])
        if self.q2_network:
            yield self.fused_loss(closs[1])
        if batch_idx % self.delayed_policy_update == 0:
            aloss = self._actor_step(training_batch, self._fill)
            yield self.fused_loss(aloss[0])
            yield self.soft_update_result()
        else:
            yield None
            yield None

    def train_batch(self, training_batch: rlt.PolicyNetworkInput, batch_idx: int = 0,
                    process_group=None, importance_weights: Optional[torch.Tensor] = None):
        """Fast path; Polyak updates fused into the Adam launches on policy-update batches.
        `importance_weights` ([B] fp32 on the batch's device, prioritized replay): each critic
        loss becomes mean_b(w_b * (q_b - y_b)^2); the actor loss stays unweighted."""
        upd = batch_idx % self.delayed_policy_update == 0
        closs = self._critic_step(training_batch, self.actor_network_target,
                                  self.q1_network_target, self.q2_network_target, self._fill,
                                  sample_weight=importance_weights)
        self.adam_step(self.q1_network.arena, process_group, polyak=upd)
        if self.q2_network:
            self.adam_step(self.q2_network.arena, process_group, polyak=upd)
        aloss = None
        if upd:
            aloss = self._actor_step(training_batch, self._fill)
            self.adam_step(self.actor_network.arena, process_group)
        self.all_batches_processed += 1
        return closs, aloss
