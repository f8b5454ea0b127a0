"""PPOTrainer (reagent/training/ppo_trainer.py:188-617): the clipped-surrogate PPO, with an
optional value net that gives either a reward-to-go baseline or the one-step TD-error
advantage.  Manual optimization as in the reference: `training_step` buffers trajectories,
`update_model` draws the reference's CPU `torch.randperm` once per epoch and runs one
`_update_model` per minibatch of trajectories.

`_update_model` packs the minibatch's trajectories and runs the fused update of
policy_gradient.py over all their rows at once -- one policy forward, the value forwards on
state (and on next_state in TD mode), one rb200_pg_returns and one rb200_pg_head launch, the
backwards -- then the value net's Adam step and the policy's.  The reference runs a separate
forward and loss graph per trajectory (:547-550).  The logger-only `_eval_metrics` is not
ported: this package has no logger.
"""
from typing import Dict, List, Optional, Union

import torch

from .. import _lib
from ..core import types as rlt
from ..optimizer import Optimizer__Union
from .policy_gradient import PolicyGradientStep, check_policy, net_grads, pack
from .reagent_lightning_module import ReAgentLightningModule


class PPOTrainer(ReAgentLightningModule):
    def __init__(
        self,
        policy,
        gamma: float = 0.9,
        optimizer: Optional[Optimizer__Union] = None,
        optimizer_value_net: Optional[Optimizer__Union] = None,
        actions: Optional[List[str]] = None,
        reward_clip: float = 1e6,
        normalize: bool = True,
        subtract_mean: bool = True,
        offset_clamp_min: bool = False,
        update_freq: int = 1,
        update_epochs: int = 1,
        ppo_batch_size: int = 1,
        ppo_epsilon: float = 0.2,
        entropy_weight: float = 0.0,
        value_net=None,
        td_error_advantage: bool = False,
    ):
        super().__init__(automatic_optimization=False)
        check_policy("PPOTrainer", policy, value_net)
        self.scorer = policy.scorer
        self.sampler = policy.sampler
        self.gamma = gamma
        # @resolve_defaults in the reference: default_factory fields
        self.optimizer_value_net = (Optimizer__Union.default() if optimizer_value_net is None
                                    else optimizer_value_net)
        self.actions = [] if actions is None else actions
        self.reward_clip = reward_clip
        self.normalize = normalize
        self.subtract_mean = subtract_mean
        self.offset_clamp_min = offset_clamp_min
        self.update_freq = update_freq
        self.update_epochs = update_epochs
        self.ppo_batch_size = ppo_batch_size
        self.ppo_epsilon = ppo_epsilon
        self.entropy_weight = entropy_weight
        self.optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        self.value_net = value_net
        self.td_error_advantage = td_error_advantage
        if value_net is not None:
            assert not self.normalize, (
                "Can't apply a value baseline and normalize rewards simultaneously")
        if td_error_advantage:
            assert value_net is not None, (
                "td_error_advantage requires a value_net to estimate V(s)")
        assert (ppo_epsilon >= 0) and (ppo_epsilon <= 1), "ppo_epsilon has to be in [0;1]"
        assert update_freq >= 1, "update_freq has to be >= 1"
        assert update_epochs >= 1, "update_epochs has to be >= 1"
        assert ppo_batch_size >= 1, "ppo_batch_size has to be >= 1"
        self.traj_buffer = []
        self._pg = PolicyGradientStep(self.scorer, self.value_net)
        self.last_losses = None

    def _check_input(self, trajectory: rlt.PolicyGradientInput) -> None:
        """:316-354, shape checks only (no synchronisation)."""
        assert trajectory.action.ndim == 2, f"action must be 2-D, got {trajectory.action.shape}"
        T = trajectory.action.shape[0]
        assert T > 0, "trajectory must contain at least one step"
        assert trajectory.reward.ndim == 1, f"reward must be 1-D, got {trajectory.reward.shape}"
        assert trajectory.log_prob.ndim == 1, f"log_prob must be 1-D, got {trajectory.log_prob.shape}"
        assert trajectory.reward.shape[0] == T, (
            f"reward length {trajectory.reward.shape[0]} != action length {T}")
        assert trajectory.log_prob.shape[0] == T, (
            f"log_prob length {trajectory.log_prob.shape[0]} != action length {T}")
        m = trajectory.possible_actions_mask
        if m is not None:
            assert m.ndim == 2, f"possible_actions_mask must be 2-D, got {m.shape}"
            assert m.shape[0] == T, f"possible_actions_mask length {m.shape[0]} != action length {T}"
        nt = trajectory.not_terminal
        if nt is not None:
            assert nt.ndim == 1, f"not_terminal must be 1-D, got {nt.shape}"
            assert nt.shape[0] == T, f"not_terminal length {nt.shape[0]} != action length {T}"
        if trajectory.next_state is not None:
            n = trajectory.next_state.float_features.shape[0]
            assert n == T, f"next_state length {n} != action length {T}"

    def _assert_final_step_terminal(self, trajectory: rlt.PolicyGradientInput) -> None:
        """:446-458: without next_state the final transition cannot bootstrap, so an explicit
        not_terminal must end in 0 (a host-syncing read, as in the reference)."""
        assert trajectory.not_terminal is None or bool(trajectory.not_terminal[-1] == 0), (
            "a truncated final transition (not_terminal[-1] != 0) needs next_state "
            "(and value_net) to bootstrap V(s_T); pass next_state or mark the last "
            "step terminal")

    def configure_optimizers(self):
        """[value net,] policy -- :490-504."""
        optimizers = []
        if self.value_net is not None:
            optimizers.append(
                self.optimizer_value_net.make_optimizer_scheduler(self.value_net.parameters()))
        optimizers.append(self.optimizer.make_optimizer_scheduler(self.scorer.parameters()))
        return optimizers

    def get_optimizers(self):
        opts = self.optimizers()
        if self.value_net is not None:
            return opts[0], opts[1]
        return None, opts[0]

    def training_step(self, training_batch: Union[rlt.PolicyGradientInput, Dict[str, torch.Tensor]],
                      batch_idx: int, optimizer_idx: int = 0):
        if isinstance(training_batch, dict):
            training_batch = rlt.PolicyGradientInput.from_dict(training_batch)
        self.traj_buffer.append(training_batch)
        if len(self.traj_buffer) == self.update_freq:
            self.update_model()

    def update_model(self):
        """:526-538: per epoch one CPU torch.randperm over the buffer, then the minibatches of
        ppo_batch_size trajectories in that order."""
        assert len(self.traj_buffer) == self.update_freq, (
            "trajectory buffer does not have sufficient samples for model_update")
        for _ in range(self.update_epochs):
            random_order = torch.randperm(len(self.traj_buffer))
            for i in range(0, len(self.traj_buffer), self.ppo_batch_size):
                idx = random_order[i: i + self.ppo_batch_size]
                self._update_model([self.traj_buffer[i] for i in idx])
        self.traj_buffer = []

    def _losses(self, trajs: List[rlt.PolicyGradientInput], do_backward: bool = True):
        """The fused losses of one minibatch: the [2] device tensor (ppo_loss summed over the
        trajectories, value_net_loss summed likewise)."""
        td = self._td()
        for t in trajs:
            self._check_input(t)
            if td and t.next_state is None:
                self._assert_final_step_terminal(t)
        p, pins = self._pack(trajs)
        return self._pg.run(p, pins, do_backward=do_backward, **self._settings(p))

    def _td(self) -> bool:
        return self.value_net is not None and self.td_error_advantage

    def _pack(self, trajs: List[rlt.PolicyGradientInput]):
        return pack(trajs, type(self).__name__, self.scorer, log_prob=True, td=self._td())

    def _settings(self, p) -> dict:
        """The fused update's settings (PolicyGradientStep.run); `p` is unused, as PPO's value
        loss is a sum."""
        if self.normalize:
            norm = _lib.PG_NORM_WHITEN if self.subtract_mean else _lib.PG_NORM_WHITEN_NO_MEAN
        else:
            norm = _lib.PG_NORM_NONE
        return dict(loss_kind=_lib.PG_LOSS_PPO, norm=norm, offset_clamp_min=self.offset_clamp_min,
                    td=self._td(), gamma=self.gamma, reward_clip=self.reward_clip,
                    temperature=self.sampler.temperature, value_scale=1.0,
                    ppo_epsilon=self.ppo_epsilon, entropy_weight=self.entropy_weight)

    def _update_model(self, training_batch_list: List[rlt.PolicyGradientInput]):
        """:540-573: the losses of every trajectory of the minibatch from the same parameters,
        then the value net's Adam step and the policy's."""
        loss = self._losses(training_batch_list)
        if self.value_net is not None:
            self.adam_step(self.value_net.arena)
        self.adam_step(self.scorer.arena)
        self.last_losses = loss
        if self.has_real_reporter:
            self.reporter.log(
                ppo_loss=loss[0].detach().reshape(1).clone(),
                value_net_loss=(loss[1].detach().reshape(1).clone() if self.value_net is not None
                                else torch.zeros(1)))

    # inspection / tests
    def advantage(self, rows: int) -> torch.Tensor:
        return self._pg.advantage(rows)

    def returns(self, rows: int) -> torch.Tensor:
        return self._pg.returns(rows)

    def net_grads(self, net):
        return net_grads(net)
