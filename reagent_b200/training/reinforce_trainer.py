"""ReinforceTrainer (reagent/training/reinforce_trainer.py:22-161): REINFORCE on one trajectory
per batch, with an optional learned baseline, on the fused update of policy_gradient.py:

  rb200_mlp_forward      policy scores [and V(state)], activations saved    :96-104, :119
  rb200_pg_returns       discounted_returns, whiten / mean subtraction, clamp  :106-116
  rb200_pg_head          eligibility, loss, d loss / d scores [, d MSE / d V]  :117-132
  rb200_mlp_backward + rb200_mlp_wgrad, per network

`train_step_gen` yields the value loss (with a value net), then the policy loss.  `train_batch`
runs the same launches and the Adam steps without a host synchronisation.
"""
import math
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..optimizer import Optimizer__Union
from .policy_gradient import PolicyGradientStep, check_policy, net_grads, pack
from .reagent_lightning_module import ReAgentLightningModule


class ReinforceTrainer(ReAgentLightningModule):
    def __init__(
        self,
        policy,
        gamma: float = 0.0,
        optimizer: Optional[Optimizer__Union] = None,
        optimizer_value_net: Optional[Optimizer__Union] = None,
        actions: Optional[List[str]] = None,
        off_policy: bool = False,
        reward_clip: float = 1e6,
        clip_param: float = 1e6,
        normalize: bool = True,
        subtract_mean: bool = True,
        offset_clamp_min: bool = False,
        value_net=None,
        do_log_metrics: bool = False,
    ):
        super().__init__()
        check_policy("ReinforceTrainer", policy, value_net)
        if do_log_metrics:
            raise NotImplementedError(
                "ReinforceTrainer: do_log_metrics needs a logger, which reagent_b200 does not have")
        # field(default_factory=...) in the reference
        self._actions = [] if actions is None else actions
        self.scorer = policy.scorer
        self.sampler = policy.sampler
        self.gamma = gamma
        self.off_policy = off_policy
        self.reward_clip = reward_clip
        self.clip_param = clip_param
        self.normalize = normalize
        self.subtract_mean = subtract_mean
        self.offset_clamp_min = offset_clamp_min
        self.optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        self.optimizer_value_net = (Optimizer__Union.default() if optimizer_value_net is None
                                    else optimizer_value_net)
        if value_net is not None:
            if self.normalize or self.subtract_mean:
                raise RuntimeError(
                    "Can't apply a baseline and reward normalization \
                    (or mean subtraction) simultaneously."
                )
            self.value_net = value_net
        else:
            self.value_net = None
        self.do_log_metrics = do_log_metrics
        self._pg = PolicyGradientStep(self.scorer, self.value_net)

    def _check_input(self, training_batch: rlt.PolicyGradientInput):
        assert training_batch.reward.ndim == 1
        if self.off_policy:
            assert training_batch.log_prob.ndim == 1

    def configure_optimizers(self):
        """[value net,] policy -- :76-90."""
        optimizers = []
        if self.value_net is not None:
            optimizers.append(
                self.optimizer_value_net.make_optimizer_scheduler(self.value_net.parameters()))
        optimizers.append(self.optimizer.make_optimizer_scheduler(self.scorer.parameters()))
        return optimizers

    def _norm(self) -> int:
        if self.normalize:
            return _lib.PG_NORM_WHITEN if self.subtract_mean else _lib.PG_NORM_WHITEN_NO_MEAN
        return _lib.PG_NORM_SUBTRACT_MEAN if self.subtract_mean else _lib.PG_NORM_NONE

    def _pack(self, batch: rlt.PolicyGradientInput):
        return pack([batch], type(self).__name__, self.scorer, log_prob=self.off_policy, td=False)

    def _settings(self, p) -> dict:
        """The fused update's settings for the packed batch `p` (PolicyGradientStep.run)."""
        return dict(loss_kind=_lib.PG_LOSS_REINFORCE, norm=self._norm(),
                    offset_clamp_min=self.offset_clamp_min, td=False, gamma=self.gamma,
                    reward_clip=self.reward_clip, temperature=self.sampler.temperature,
                    value_scale=1.0 / p.rows, log_clip_param=math.log(float(self.clip_param)))

    def _step(self, batch: rlt.PolicyGradientInput, do_backward: bool = True) -> torch.Tensor:
        """The update's launches.  Returns the [2] device tensor (policy loss, value loss)."""
        p, pins = self._pack(batch)
        return self._pg.run(p, pins, do_backward=do_backward, **self._settings(p))

    def train_step_gen(self, training_batch: rlt.PolicyGradientInput, batch_idx: int):
        """Yields [the value loss,] the policy loss -- :92-148."""
        self._check_input(training_batch)
        loss = self._step(training_batch)
        if self.value_net is not None:
            yield self.fused_loss(loss[1])
        yield self.fused_loss(loss[0])

    def train_batch(self, training_batch: rlt.PolicyGradientInput, batch_idx: int = 0,
                    process_group=None):
        """Fast path: the update of train_step_gen and its Adam steps, with no host
        synchronisation and without _check_input.  Returns the [2] device tensor (policy loss,
        value loss)."""
        loss = self._step(training_batch)
        if self.value_net is not None:
            self.adam_step(self.value_net.arena, process_group)
        self.adam_step(self.scorer.arena, process_group)
        self.all_batches_processed += 1
        return loss

    # inspection / tests
    def advantage(self, rows: int) -> torch.Tensor:
        return self._pg.advantage(rows)

    def returns(self, rows: int) -> torch.Tensor:
        return self._pg.returns(rows)

    def net_grads(self, net):
        return net_grads(net)
