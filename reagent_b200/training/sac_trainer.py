"""SACTrainer with the reference's constructor, optimizer order and generator protocol
(reagent/training/sac_trainer.py:50-385): twin (or single) critics, learnable or fixed entropy
temperature, an optional state-value network and CRR weighting of the actor loss.

Launch sequence of one update (value_network=None):
  rb200_ac_critic_step  target + q1/q2 losses + critic dZ chains     sac_trainer.py:214-248
  rb200_mlp_wgrad x2, Adam(q1), Adam(q2) [+ fused Polyak]            optimizer.py / soft_update.py
  rb200_ac_actor_step   actor + alpha losses, backward through the UPDATED critics  :254-322
  rb200_mlp_wgrad, Adam(actor), Adam(log_alpha) -> entropy_temperature = exp(log_alpha)
With a value network the critic step's target is r + gamma * V'(s') (no actor forward on s',
one noise draw per update), the actor step also writes min_c q_c(s, pi(s)), and after the
alpha step rb200_ac_value_step, rb200_mlp_wgrad and Adam(value) [+ fused Polyak into the value
target] train V(s) against it (:329-343).  Only the value target is soft-updated then.
Sequential dependence of the reference is kept (SURVEY.md facts 3-4): the actor step sees the
post-update critics; the new temperature takes effect in the value step and the next batch.
"""
import copy
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import RLParameters
from ..models.arena import ScalarArena
from ..optimizer import Optimizer__Union, SoftUpdate
from .actor_critic_base import ActorCriticBase
from .workspace import Pins, batch_device, wgrad

_DEFAULT = object()


@dataclass
class CRRWeightFn:
    """Critic Regularized Regression weight of the advantage (sac_trainer.py:23-48): the
    indicator advantage >= indicator_fn_threshold, or exp(advantage / exponent_beta), clamped
    to [0, exponent_clamp] when exponent_clamp is set."""
    indicator_fn_threshold: Optional[float] = None
    exponent_beta: Optional[float] = None
    exponent_clamp: Optional[float] = None

    def __post_init__(self):
        assert self.exponent_beta or self.indicator_fn_threshold
        assert not (self.exponent_beta and self.indicator_fn_threshold)
        if self.exponent_beta:
            assert self.exponent_beta > 1e-6
        if self.exponent_clamp:
            assert self.exponent_clamp > 1e-6

    def get_weight_from_advantage(self, advantage):
        if self.indicator_fn_threshold:
            return (advantage >= self.indicator_fn_threshold).float()
        if self.exponent_beta:
            exp = torch.exp(advantage / self.exponent_beta)
            if self.exponent_clamp:
                exp = torch.clamp(exp, 0.0, self.exponent_clamp)
            return exp

    def fill(self, a):
        """The kernels' CRR fields of rb200_ac_args_t."""
        if self.indicator_fn_threshold:
            a.crr_mode = _lib.CRR_INDICATOR
            a.crr_threshold = float(self.indicator_fn_threshold)
        else:
            a.crr_mode = _lib.CRR_EXPONENT
            a.crr_beta = float(self.exponent_beta)
            a.crr_clamp = float(self.exponent_clamp) if self.exponent_clamp else 0.0


class SACTrainer(ActorCriticBase):
    ALGO = _lib.ALGO_SAC

    def __init__(
        self,
        actor_network,
        q1_network,
        q2_network=None,
        value_network=None,
        rl: Optional[RLParameters] = None,
        q_network_optimizer: Optional[Optimizer__Union] = None,
        value_network_optimizer: Optional[Optimizer__Union] = None,
        actor_network_optimizer: Optional[Optimizer__Union] = None,
        alpha_optimizer=_DEFAULT,
        minibatch_size: int = 1024,
        entropy_temperature: float = 0.01,
        logged_action_uniform_prior: bool = True,
        target_entropy: float = -1.0,
        action_embedding_kld_weight: Optional[float] = None,
        apply_kld_on_mean: bool = False,
        action_embedding_mean: Optional[List[float]] = None,
        action_embedding_variance: Optional[List[float]] = None,
        crr_config=None,
        backprop_through_log_prob: bool = True,
    ) -> None:
        super().__init__()
        self._ac_init()
        if action_embedding_kld_weight:
            raise NotImplementedError("action-embedding KLD is out of scope")
        if crr_config is not None:
            assert value_network is not None  # sac_trainer.py:142-144
            if not backprop_through_log_prob:
                # the CRR loss -clamp(log_prob) * w has no other path to the actor
                raise ValueError("crr_config needs backprop_through_log_prob=True: without it "
                                 "the actor loss has no gradient")
        self.rl_parameters = RLParameters() if rl is None else rl
        self.q1_network = q1_network
        self.q2_network = q2_network
        self.q_network_optimizer = q_network_optimizer or Optimizer__Union.default()
        self.value_network = value_network
        self.value_network_optimizer = value_network_optimizer or Optimizer__Union.default()
        if self.value_network is not None:
            self.value_network_target = copy.deepcopy(self.value_network)
        else:
            self.q1_network_target = copy.deepcopy(self.q1_network)
            self.q2_network_target = copy.deepcopy(self.q2_network)
        self.actor_network = actor_network
        self.actor_network_optimizer = actor_network_optimizer or Optimizer__Union.default()
        self.entropy_temperature = entropy_temperature
        self.alpha_optimizer = (Optimizer__Union.default() if alpha_optimizer is _DEFAULT
                                else alpha_optimizer)
        if self.alpha_optimizer is not None:
            self.target_entropy = target_entropy
            # the reference keeps log_alpha in float64 (np.log -> torch.tensor); the fused Adam
            # is fp32 -- the difference is ~1e-8 relative, far inside the parity tolerance
            self.log_alpha = torch.nn.Parameter(
                torch.tensor([np.log(self.entropy_temperature)], dtype=torch.float32))
        else:
            self.target_entropy = target_entropy
        # not part of the state_dict (the reference has no such key): re-derived from log_alpha
        self.register_buffer("_alpha_dev", torch.tensor([float(entropy_temperature)]),
                             persistent=False)
        self.register_load_state_dict_post_hook(SACTrainer._rederive_alpha)
        self.logged_action_uniform_prior = logged_action_uniform_prior
        self.add_kld_to_loss = False
        self.crr_config = crr_config
        self.backprop_through_log_prob = backprop_through_log_prob
        self.minibatch_size = minibatch_size

    @staticmethod
    def _rederive_alpha(module, incompatible_keys):
        if module.alpha_optimizer is not None:  # sac_trainer.py:322
            with torch.no_grad():
                module._alpha_dev.copy_(module.log_alpha.data.exp().to(module._alpha_dev.device))
            module.entropy_temperature = module._alpha_dev

    def configure_optimizers(self):
        """q1, q2, actor, alpha, value, SoftUpdate (sac_trainer.py:148-193)."""
        optimizers = []
        optimizers.append(
            self.q_network_optimizer.make_optimizer_scheduler(self.q1_network.parameters()))
        if self.q2_network:
            optimizers.append(
                self.q_network_optimizer.make_optimizer_scheduler(self.q2_network.parameters()))
        optimizers.append(
            self.actor_network_optimizer.make_optimizer_scheduler(
                self.actor_network.parameters()))
        if self.alpha_optimizer is not None:
            optimizers.append(self.alpha_optimizer.make_optimizer_scheduler([self.log_alpha]))
        if self.value_network:
            optimizers.append(self.value_network_optimizer.make_optimizer_scheduler(
                self.value_network.parameters()))
            target_params = list(self.value_network_target.parameters())
            source_params = list(self.value_network.parameters())
        else:
            target_params = list(self.q1_network_target.parameters())
            source_params = list(self.q1_network.parameters())
            if self.q2_network:
                target_params += list(self.q2_network_target.parameters())
                source_params += list(self.q2_network.parameters())
        optimizers.append(
            SoftUpdate.make_optimizer_scheduler(target_params, source_params, tau=self.tau))
        return optimizers

    # ---- kernel argument fillers --------------------------------------------------
    def _fill_critic(self, a, pins):
        dev = self._ws["dev"]
        if self._alpha_dev.device != dev:  # trainer built from CUDA networks, never .cuda()'d
            self._alpha_dev = self._alpha_dev.to(dev)
            if self.alpha_optimizer is not None and self.log_alpha.device != dev:
                raise _lib.Rb200Error("SACTrainer: log_alpha is not on the networks' device -- "
                                      "move the trainer with .cuda()/.to(device) before "
                                      "configure_optimizers()")
        a.alpha = _lib.ptr(self._alpha_dev, dev)
        a.target_entropy = float(self.target_entropy)
        a.backprop_through_log_prob = int(bool(self.backprop_through_log_prob))
        if self.value_network is not None:
            a.value_target = self._desc_ptr(self.value_network_target, pins)

    def _fill_actor(self, a, pins):
        self._fill_critic(a, pins)
        ws = self._ws
        A = self.q1_network.arena.dims[0] - self.actor_network.arena.dims[0]
        a.noise_cur = self._noise("cur", ws["B"], A, pins)
        if self.alpha_optimizer is not None:
            a.alpha_grad = ws["alpha_grad"].data_ptr()
            a.log_alpha = _lib.ptr(self.log_alpha.data, ws["dev"])
        if self.value_network is not None:
            a.value_target = None
            a.min_q_out = ws["min_q"].data_ptr()
            if self.crr_config is not None:
                a.value_net = self._desc_ptr(self.value_network, pins)
                self.crr_config.fill(a)

    @staticmethod
    def _desc_ptr(net, pins):
        d = net.arena.desc()
        pins.keep.append(d)
        return _lib.C.pointer(d)

    def _value_step(self, batch):
        """V(s) against min_q (minus alpha * clamp(log_prob) without the uniform prior), with
        the log-probs and min-of-critics the actor step of this update wrote
        (sac_trainer.py:329-343), then V's weight gradients."""
        B = batch.state.float_features.shape[0]
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        ws = self._workspace(B, pins.device)
        a, state = self._value_args(batch, ws, pins)
        rc = _lib.lib().rb200_ac_value_step(self._desc(self.value_network), a, ws["value"].c,
                                            _lib.cur_stream())
        _lib.check(rc, "rb200_ac_value_step")
        wgrad(self.value_network.arena, ws["value"], state, B)
        return ws["value_loss"]

    def _value_args(self, batch, ws, pins):
        """(args, state) of rb200_ac_value_step on workspace `ws`, as _base_args."""
        a, state = self._base_args(batch, ws, pins)
        a.loss = ws["value_loss"].data_ptr()
        a.min_q_out = ws["min_q"].data_ptr()
        a.log_prob_out = ws["log_prob"].data_ptr()
        a.alpha = _lib.ptr(self._alpha_dev, ws["dev"])
        a.logged_action_uniform_prior = int(bool(self.logged_action_uniform_prior))
        return a, state

    def _critic_targets(self):
        if self.value_network is not None:
            return None, None
        return self.q1_network_target, self.q2_network_target

    def _alpha_arena(self):
        arena = getattr(self.log_alpha, "_rb200_arena", None)
        if arena is None:
            arena = ScalarArena(self.log_alpha)
        return arena

    # ---- reference protocol -----------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.PolicyNetworkInput, batch_idx: int):
        """IMPORTANT: the input action is assumed to match the actor's output range."""
        assert isinstance(training_batch, rlt.PolicyNetworkInput)
        closs = self._critic_step(training_batch, self.actor_network, *self._critic_targets(),
                                  self._fill_critic)
        yield self.fused_loss(closs[0])
        if self.q2_network:
            yield self.fused_loss(closs[1])
        aloss = self._actor_step(training_batch, self._fill_actor)
        yield self.fused_loss(aloss[0])
        if self.alpha_optimizer is not None:
            arena = self._alpha_arena()
            arena.gpart = self._ws["alpha_grad"]
            arena.grad_ready = True
            yield self.fused_loss(aloss[1])
            # sac_trainer.py:322 (runs after the alpha step, used from the next batch on)
            self._alpha_dev.copy_(self.log_alpha.data.exp())
            self.entropy_temperature = self._alpha_dev
        if self.value_network is not None:
            yield self.fused_loss(self._value_step(training_batch)[0])
        if self.logger:
            self.logger.log_metrics(
                {"td_loss": closs[0], "q1_value": self._ws["q1_value"].mean(),
                 "entropy_temperature": self.entropy_temperature,
                 "target_q_value": self._ws["td_target"].mean(), "actor_loss": aloss[0]},
                step=self.all_batches_processed)
        result = self.soft_update_result()
        self.log("td_loss", closs[0], prog_bar=True)
        yield result

    def train_batch(self, training_batch: rlt.PolicyNetworkInput, batch_idx: int = 0,
                    process_group=None, importance_weights: Optional[torch.Tensor] = None):
        """Fast path: the whole update (same arithmetic as train_step_gen), Polyak updates
        fused into the critics' Adam launches, exp(log_alpha) into the alpha launch.
        `importance_weights` ([B] fp32 on the batch's device, prioritized replay): each critic
        loss becomes mean_b(w_b * (q_b - y_b)^2); the actor, alpha and value losses stay
        unweighted."""
        opts = self.optimizers()
        i = 0
        q1t, q2t = self._critic_targets()
        closs = self._critic_step(training_batch, self.actor_network, q1t, q2t,
                                  self._fill_critic, sample_weight=importance_weights)
        self._dp_step(opts[i], self.q1_network.arena, None if q1t is None else q1t.arena,
                      process_group)
        i += 1
        if self.q2_network:
            self._dp_step(opts[i], self.q2_network.arena, None if q2t is None else q2t.arena,
                          process_group)
            i += 1
        aloss = self._actor_step(training_batch, self._fill_actor)
        self._dp_step(opts[i], self.actor_network.arena, None, process_group)
        i += 1
        if self.alpha_optimizer is not None:
            arena = self._alpha_arena()
            arena.gpart = self._ws["alpha_grad"]
            arena.grad_ready = True
            self._dp_step(opts[i], arena, None, process_group, exp_out=self._alpha_dev)
            self.entropy_temperature = self._alpha_dev
            i += 1
        if self.value_network is not None:
            self._value_step(training_batch)
            self._dp_step(opts[i], self.value_network.arena, self.value_network_target.arena,
                          process_group)
        self.all_batches_processed += 1
        return closs, aloss

    def _dp_step(self, opt, arena, target, process_group, exp_out=None):
        from .data_parallel import dp_fused_step

        dp_fused_step(opt, arena, process_group, target=target, tau=self.tau, exp_out=exp_out)
