"""DQNTrainerMixin / DQNTrainerBaseLightning: the parts of
reagent/training/dqn_trainer_base.py:23-452 that are on the hot path, including the CPE
heads (reward network, q_network_cpe, `_calculate_cpes`, :243-452): two extra MLPs evaluated
by the generic forward / backward / weight-gradient kernels with rb200_cpe_heads in between,
and the counterfactual policy evaluation they feed (gather_eval_data / validation_epoch_end,
:454-509): EvaluationDataPages reduced by the Evaluator of reagent_b200.evaluation."""
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import EvaluationParameters, RLParameters
from .reagent_lightning_module import ReAgentLightningModule
from .rl_trainer_pytorch import RLTrainerMixin
from .workspace import (NetWorkspace, Pins, backward_wgrad, batch_device, discount_source,
                        loss_kind, register_reward_boosts, ws_fits)


class DQNTrainerMixin:
    ACTION_NOT_POSSIBLE_VAL = -1e9

    def get_max_q_values(self, q_values, possible_actions_mask):
        return self.get_max_q_values_with_target(q_values, q_values, possible_actions_mask)

    def get_max_q_values_with_target(self, q_values, q_values_target, possible_actions_mask):
        """Host-visible utility with the reference's semantics (dqn_trainer_base.py:33-77).
        The training path does this inside the fused TD kernel; this method exists for
        callers / logging that use it directly (tiny tensors, torch plumbing)."""
        q_values = q_values.reshape(possible_actions_mask.shape)
        q_values_target = q_values_target.reshape(possible_actions_mask.shape)
        inverse_pna = 1 - possible_actions_mask
        impossible_action_penalty = self.ACTION_NOT_POSSIBLE_VAL * inverse_pna
        q_values = q_values + impossible_action_penalty
        q_values_target = q_values_target + impossible_action_penalty
        if self.double_q_learning:
            max_q_values, max_indicies = torch.max(q_values, dim=1, keepdim=True)
            max_q_values_target = torch.gather(q_values_target, 1, max_indicies)
        else:
            max_q_values_target, max_indicies = torch.max(q_values_target, dim=1, keepdim=True)
        return max_q_values_target, max_indicies


class DQNTrainerBaseLightning(DQNTrainerMixin, RLTrainerMixin, ReAgentLightningModule):
    def __init__(
        self,
        rl_parameters: RLParameters,
        metrics_to_score=None,
        actions: Optional[List[str]] = None,
        evaluation_parameters: Optional[EvaluationParameters] = None,
    ):
        super().__init__()
        self.rl_parameters = rl_parameters
        self.time_diff_unit_length = rl_parameters.time_diff_unit_length
        self.tensorboard_logging_freq = rl_parameters.tensorboard_logging_freq
        self.calc_cpe_in_training = bool(
            evaluation_parameters and evaluation_parameters.calc_cpe_in_training)
        assert actions is not None
        self._actions: List[str] = actions
        self.q_network_loss_kind = loss_kind(rl_parameters.q_network_loss)
        if metrics_to_score:
            self.metrics_to_score = metrics_to_score + ["reward"]
        else:
            self.metrics_to_score = ["reward"]
        register_reward_boosts(self, self._actions, rl_parameters.reward_boost)
        # mirror of the reference's host-syncing `.any()` input check; off by default
        self.strict_input_checks = False

    def _initialize_cpe(self, reward_network, q_network_cpe, q_network_cpe_target, optimizer):
        """dqn_trainer_base.py:243-311: store the reward / CPE networks, the offsets of every
        metric's block of `num_actions` outputs, and the Evaluator that validation_epoch_end
        runs on the pages of validation_step."""
        self._cpe_ws = None
        if not self.calc_cpe_in_training:
            self.reward_network = None
            self.q_network_cpe = None
            self.q_network_cpe_target = None
            return
        assert reward_network is not None, "reward_network is required for CPE"
        assert q_network_cpe is not None and q_network_cpe_target is not None, (
            "q_network_cpe and q_network_cpe_target are required for CPE")
        self.reward_network = reward_network
        self.reward_network_optimizer = optimizer
        self.q_network_cpe = q_network_cpe
        self.q_network_cpe_target = q_network_cpe_target
        self.q_network_cpe_optimizer = optimizer
        num_output_nodes = len(self.metrics_to_score) * self.num_actions
        self.register_buffer("reward_idx_offsets",
                             torch.arange(0, num_output_nodes, self.num_actions, dtype=torch.long))
        from ..evaluation.evaluator import Evaluator

        reward_stripped = self.metrics_to_score[:-1] if len(self.metrics_to_score) > 1 else None
        self.evaluator = Evaluator(self._actions, self.rl_parameters.gamma, self,
                                   metrics_to_score=reward_stripped)

    def page_model_outputs(self, state):
        """The model outputs an EvaluationDataPage scores the policy with (the first element of
        get_detached_model_outputs: q_network for DQN, the actor for CRR)."""
        return self.get_detached_model_outputs(state)[0]

    def gather_eval_data(self, validation_step_outputs):
        """Concatenate the EvaluationDataPages of validation_step, then sort, compute_values and
        validate when the pages carry mdp_id (:454-486).  The pages stay on their device."""
        eval_data = None
        for edp in validation_step_outputs:
            eval_data = edp if eval_data is None else eval_data.append(edp)
        if eval_data and eval_data.mdp_id is not None:
            eval_data = eval_data.sort()
            eval_data = eval_data.compute_values(self.gamma)
            eval_data.validate()
        return eval_data

    def validation_epoch_end(self, valid_step_outputs):
        """Run the Evaluator on the gathered pages and log its CpeDetails (:498-509)."""
        eval_data = self.gather_eval_data(valid_step_outputs)
        if eval_data and eval_data.mdp_id is not None:
            cpe_details = self.evaluator.evaluate_post_training(eval_data)
            self.reporter.log(cpe_details=cpe_details)

    def _configure_cpe_optimizers(self):
        """(target params, source params, [reward optimizer, cpe optimizer]) -- :313-330."""
        target_params = list(self.q_network_cpe_target.parameters())
        source_params = list(self.q_network_cpe.parameters())
        optimizers = [
            self.reward_network_optimizer.make_optimizer_scheduler(self.reward_network.parameters()),
            self.q_network_cpe_optimizer.make_optimizer_scheduler(self.q_network_cpe.parameters()),
        ]
        return target_params, source_params, optimizers

    def _cpe_workspace(self, B: int, device):
        if not ws_fits(self._cpe_ws, B, device):
            MA = len(self.metrics_to_score) * self.num_actions
            self._cpe_ws = {
                "B": B, "dev": device,
                "reward": NetWorkspace(self.reward_network.arena, B, device),
                "qcpe": NetWorkspace(self.q_network_cpe.arena, B, device),
                "next_scores": torch.empty(B, self.num_actions, device=device),
                "reward_est": torch.empty(B, MA, device=device),
                "qcpe_out": torch.empty(B, MA, device=device),
                "qcpe_t_next": torch.empty(B, MA, device=device),
                "prop_next": torch.empty(B, self.num_actions, device=device),
                "loss_partials": torch.zeros(2 * ((B + 255) // 256), device=device),
                "loss": torch.zeros(2, device=device),
                "counter": torch.zeros(1, dtype=torch.int32, device=device),
            }
        return self._cpe_ws

    def _calculate_cpes(self, training_batch: rlt.DiscreteDqnInput,
                        next_actions_mask: Optional[torch.Tensor] = None,
                        next_scores: Optional[torch.Tensor] = None,
                        constant_discount: bool = False):
        """_calculate_cpes (:332-452) on the device: returns the [2] loss tensor (reward loss,
        CPE q-value loss) and leaves the gradient partials of both networks in their arenas.
        Runs AFTER the q-network step of the same batch, as in the reference's generator
        (all_next_action_scores is evaluated after `yield td_loss`, dqn_trainer.py:266-268).
        `next_actions_mask` replaces the batch's next-action mask of the model propensities
        (DQNTrainer with BCQ passes its filtered mask).  `next_scores` ([B, A] fp32 on the
        batch's device) are the next-state scores the propensities come from, in place of a
        forward of q_network on next_state; `constant_discount` discounts by gamma whatever the
        batch's time_diff / step say.  DiscreteCRRTrainer passes q1_network_target(next_state)
        from before its critic steps and a constant gamma (discrete_crr_trainer.py:308-367)."""
        pins = Pins(batch_device(training_batch.state.float_features, type(self).__name__))
        state = pins.tensor(training_batch.state.float_features)
        next_state = pins.tensor(training_batch.next_state.float_features)
        B = state.shape[0]
        ws = self._cpe_workspace(B, pins.device)

        def fwd(net, x, out, save=None):
            net.arena.refresh()
            net.arena.forward(x, out, save=save)

        if next_scores is None:
            fwd(self.q_network, next_state, ws["next_scores"])
            next_scores = ws["next_scores"]
        fwd(self.reward_network, state, ws["reward_est"], ws["reward"])
        fwd(self.q_network_cpe, state, ws["qcpe_out"], ws["qcpe"])
        fwd(self.q_network_cpe_target, next_state, ws["qcpe_t_next"])
        metrics = training_batch.extras.metrics if training_batch.extras is not None else None
        mrc = training_batch.reward if metrics is None else torch.cat((training_batch.reward, metrics), dim=1)
        M = len(self.metrics_to_score)
        assert mrc.shape[1] == M, f"reward + metrics have {mrc.shape[1]} columns, metrics_to_score {M}"
        a = _lib.CpeArgsT()
        a.batch, a.num_actions, a.num_metrics = B, self.num_actions, M
        a.next_scores = pins(next_scores)
        mask = (training_batch.possible_next_actions_mask if self.maxq_learning
                else training_batch.next_action)
        if next_actions_mask is not None:
            mask = next_actions_mask
        a.mask = pins(mask)
        a.temperature = float(self.rl_temperature)
        a.action = pins(training_batch.action)
        a.metrics_reward = pins(mrc)
        a.gamma = float(self.gamma)
        src = None if constant_discount else discount_source(self, training_batch)
        a.discount_src = pins(src)
        a.discount_mode = _lib.DISCOUNT_CONST if src is None else _lib.DISCOUNT_POW
        a.not_terminal = pins(training_batch.not_terminal.reshape(-1))
        a.reward_est = ws["reward_est"].data_ptr()
        a.qcpe = ws["qcpe_out"].data_ptr()
        a.qcpe_target_next = ws["qcpe_t_next"].data_ptr()
        a.loss_kind = self.q_network_loss_kind
        Lr, Lc = len(self.reward_network.arena.acts), len(self.q_network_cpe.arena.acts)
        a.dz_reward = ws["reward"].dz[Lr - 1].data_ptr()
        a.dz_qcpe = ws["qcpe"].dz[Lc - 1].data_ptr()
        a.propensities_next = ws["prop_next"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        _lib.check(_lib.lib().rb200_cpe_heads(a, _lib.cur_stream()), "rb200_cpe_heads")
        for net, w in ((self.reward_network, ws["reward"]), (self.q_network_cpe, ws["qcpe"])):
            backward_wgrad(net.arena, w, state, B)
            net.arena.finish_grads()
        self.model_propensities_next_states = ws["prop_next"]
        return ws["loss"]

    def _check_input(self, training_batch: rlt.DiscreteDqnInput):
        assert isinstance(training_batch, rlt.DiscreteDqnInput)
        assert training_batch.not_terminal.dim() == training_batch.reward.dim() == 2
        assert training_batch.not_terminal.shape[1] == training_batch.reward.shape[1] == 1
        assert training_batch.action.dim() == training_batch.next_action.dim() == 2
        assert (training_batch.action.shape[1] == training_batch.next_action.shape[1]
                == self.num_actions)
        if self.strict_input_checks and training_batch.possible_next_actions_mask is not None:
            if torch.logical_and(
                training_batch.possible_next_actions_mask.float().sum(dim=1) == 0,
                training_batch.not_terminal.squeeze().bool(),
            ).any():
                raise ValueError(
                    "No possible next actions. Should the environment have terminated?")

    @property
    def num_actions(self) -> int:
        assert self._actions is not None, "Not a discrete action DQN"
        return len(self._actions)

    @torch.no_grad()
    def boost_rewards(self, rewards: torch.Tensor, actions: torch.Tensor) -> torch.Tensor:
        """Utility with the reference's semantics (dqn_trainer_base.py:216-241); the
        training path applies the boost inside the fused kernel."""
        reward_boosts = torch.sum(actions.float() * self.reward_boosts, dim=1, keepdim=True)
        return rewards + reward_boosts
