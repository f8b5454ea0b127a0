"""DiscreteCRRTrainer: Critic Regularized Regression (https://arxiv.org/abs/2006.15134) for
discrete actions, with the reference's constructor, optimizer order and generator protocol
(reagent/training/discrete_crr_trainer.py:24-440).  Launches of one update with twin critics:

  rb200_mlp_forward x3   actor (or target actor), q1_target, q2_target on next_state    :198-212
  rb200_mlp_forward x2   q1, q2 on state, activations saved                             :214-218
  rb200_crr_critic_head  TD target, both MSE losses, d loss / d q of both critics
  rb200_mlp_backward + rb200_mlp_wgrad + Adam (Polyak folded in), per critic
  rb200_mlp_forward x2   the UPDATED q1 on state; the actor on state, activations saved  :328-332
  rb200_crr_actor_head   advantage weights, actor loss (+ entropy term), d loss / dz     :220-288
  rb200_mlp_backward + rb200_mlp_wgrad + Adam (Polyak folded in)

18 launches (13 with one critic), plus one fold / unfold pair per dueling critic use, two
draws with exploration noise, and the CPE step of DQNTrainerBaseLightning when it is on.  On a
batch where `batch_idx % delayed_policy_update != 0` the actor head and the actor's backward and
Adam are skipped (the yield is None), but every target still takes its soft update: the
reference's SoftUpdate is the last optimizer of every batch, unlike TD3Trainer's.

The actor's logits are its forward's output, FullyConnectedActor.forward (reagent/models/
actor.py:90-110): action_activation(z), and with `exploration_variance` set
clamp(action_activation(z) + noise, -1, 1), noise ~ N(0, exploration_variance) with
exploration_variance as the SCALE, drawn anew for each of the two forwards of an update, in
training too.  `noise_hook(name, shape, device)` (name "next" or "cur") replaces the N(0, 1)
draw that is then scaled, so that tests can inject the reference's draws.
"""
from typing import List, Optional, Tuple

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import EvaluationParameters, RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .dqn_trainer_base import DQNTrainerBaseLightning
from .workspace import NetWorkspace, Pins, backward_wgrad, batch_device, param_grads, ws_fits


class DiscreteCRRTrainer(DQNTrainerBaseLightning):
    def __init__(
        self,
        actor_network,
        actor_network_target,
        q1_network,
        q1_network_target,
        reward_network,
        q2_network=None,
        q2_network_target=None,
        q_network_cpe=None,
        q_network_cpe_target=None,
        metrics_to_score=None,
        evaluation: Optional[EvaluationParameters] = None,
        rl: Optional[RLParameters] = None,
        double_q_learning: bool = True,
        q_network_optimizer: Optional[Optimizer__Union] = None,
        actor_network_optimizer: Optional[Optimizer__Union] = None,
        use_target_actor: bool = False,
        actions: Optional[List[str]] = None,
        delayed_policy_update: int = 1,
        beta: float = 1.0,
        entropy_coeff: float = 0.0,
        clip_limit: float = 10.0,
        max_weight: float = 20.0,
    ) -> None:
        # @resolve_defaults in the reference (:30): default_factory fields
        evaluation = EvaluationParameters() if evaluation is None else evaluation
        rl = RLParameters() if rl is None else rl
        actions = [] if actions is None else actions
        super().__init__(rl, metrics_to_score=metrics_to_score, actions=actions,
                         evaluation_parameters=evaluation)
        self.double_q_learning = double_q_learning
        self.use_target_actor = use_target_actor
        self._check_networks(actor_network, q1_network, q2_network)
        self.q1_network = q1_network
        self.q1_network_target = q1_network_target
        self.q_network_optimizer = q_network_optimizer or Optimizer__Union.default()
        self.q2_network = q2_network
        if self.q2_network is not None:
            assert q2_network_target is not None, "q2_network provided without a target network"
            self.q2_network_target = q2_network_target
        else:
            self.q2_network_target = None
        self.actor_network = actor_network
        self.actor_network_target = actor_network_target
        self.actor_network_optimizer = actor_network_optimizer or Optimizer__Union.default()
        self.delayed_policy_update = delayed_policy_update
        self._initialize_cpe(reward_network, q_network_cpe, q_network_cpe_target,
                             optimizer=self.q_network_optimizer)
        self.beta = beta
        self.entropy_coeff = entropy_coeff
        self.clip_limit = clip_limit
        self.max_weight = max_weight
        self.noise_hook = None
        self._ws = None

    def _check_networks(self, actor, q1, q2) -> None:
        from ..models import DuelingQNetwork, FullyConnectedActor, FullyConnectedDQN

        if not isinstance(actor, FullyConnectedActor):
            raise NotImplementedError(
                "DiscreteCRRTrainer needs a reagent_b200.models.FullyConnectedActor (its forward "
                "runs on the fused MLP kernel); got " + type(actor).__name__)
        nets = [("actor_network", actor.action_dim)]
        for name, q in (("q1_network", q1), ("q2_network", q2)):
            if q is None:
                continue
            if not isinstance(q, (FullyConnectedDQN, DuelingQNetwork)) or q.num_atoms is not None:
                raise NotImplementedError(
                    f"DiscreteCRRTrainer: {name} must be a reagent_b200.models.FullyConnectedDQN "
                    "or DuelingQNetwork without atoms (one value per action from the fused MLP "
                    "kernel); got " + type(q).__name__)
            nets.append((name, q.action_dim))
        for name, n in nets:
            if n != self.num_actions:
                raise ValueError(f"{name} has {n} outputs, but there are {self.num_actions} actions")
        if self.num_actions > 1024:
            raise NotImplementedError("the CRR loss heads hold one row per warp: at most 1024 actions")

    @property
    def q_network(self):
        return self.q1_network

    @torch.no_grad()
    def get_detached_model_outputs(self, state) -> Tuple[torch.Tensor, None]:
        """The actor's scores (model propensities come from them), and None where DQNTrainer
        returns its target scores -- :144-151."""
        return self.actor_network(state).action, None

    def configure_optimizers(self):
        """q1, [q2], actor, [reward, q_cpe], SoftUpdate(q1, [q2], actor, [q_cpe]) -- :153-196."""
        optimizers = []
        target_params = list(self.q1_network_target.parameters())
        source_params = list(self.q1_network.parameters())
        optimizers.append(
            self.q_network_optimizer.make_optimizer_scheduler(self.q1_network.parameters()))
        if self.q2_network:
            target_params += list(self.q2_network_target.parameters())
            source_params += list(self.q2_network.parameters())
            optimizers.append(
                self.q_network_optimizer.make_optimizer_scheduler(self.q2_network.parameters()))
        target_params += list(self.actor_network_target.parameters())
        source_params += list(self.actor_network.parameters())
        optimizers.append(
            self.actor_network_optimizer.make_optimizer_scheduler(
                self.actor_network.parameters()))
        if self.calc_cpe_in_training:
            cpe_targets, cpe_sources, cpe_optimizers = self._configure_cpe_optimizers()
            target_params += cpe_targets
            source_params += cpe_sources
            optimizers += cpe_optimizers
        optimizers.append(
            SoftUpdate.make_optimizer_scheduler(target_params, source_params, tau=self.tau))
        return optimizers

    # ------------------------------------------------------------------
    def _workspace(self, B: int, device):
        if not ws_fits(self._ws, B, device):
            A = self.num_actions
            q2 = self.q2_network

            def ba():
                return torch.empty(B, A, device=device)

            nparts = 2 * (-(-B // _lib.CRR_ROWS_PER_BLOCK))
            self._ws = {
                "B": B, "dev": device,
                "actor": NetWorkspace(self.actor_network.arena, B, device),
                "q1": NetWorkspace(self.q1_network.arena, B, device),
                "q2": None if q2 is None else NetWorkspace(q2.arena, B, device),
                "actor_next": ba(), "q1t_next": ba(), "q2t_next": None if q2 is None else ba(),
                "q1_out": ba(), "q2_out": None if q2 is None else ba(), "actor_out": ba(),
                "td_target": torch.empty(B, device=device),
                "q1_sel": torch.empty(B, device=device), "q2_sel": torch.empty(B, device=device),
                "weight": torch.empty(B, device=device),
                "critic_partials": torch.zeros(nparts, device=device),
                "actor_partials": torch.zeros(nparts, device=device),
                "critic_loss": torch.zeros(2, device=device),
                "actor_loss": torch.zeros(2, device=device),
                "counter": torch.zeros(2, dtype=torch.int32, device=device),
            }
        return self._ws

    def _noise(self, name: str, B: int, pins: Pins) -> Optional[torch.Tensor]:
        """The exploration noise of one actor forward ([B, A], scaled), or None."""
        scale = self.actor_network.exploration_variance
        if scale is None:
            return None
        shape = (B, self.num_actions)
        z = (self.noise_hook(name, shape, pins.device) if self.noise_hook is not None
             else torch.randn(shape, device=pins.device))
        return pins.tensor(z * scale)

    @staticmethod
    def _forward(net, x, out, save=None):
        net.arena.refresh()  # no-op for plain MLPs; folds a dueling head
        net.arena.forward(x, out, save=save)

    def _critic_step(self, batch: rlt.DiscreteDqnInput, do_backward: bool = True) -> torch.Tensor:
        """Target and critic losses (and both critics' gradient partials).  Returns the [2] device
        tensor (q1 loss, q2 loss); no host synchronisation."""
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        state = pins.tensor(batch.state.float_features)
        next_state = pins.tensor(batch.next_state.float_features)
        B = state.shape[0]
        ws = self._workspace(B, pins.device)
        q2 = self.q2_network
        actor = self.actor_network_target if self.use_target_actor else self.actor_network
        self._forward(actor, next_state, ws["actor_next"])
        self._forward(self.q1_network_target, next_state, ws["q1t_next"])
        self._forward(self.q1_network, state, ws["q1_out"], ws["q1"] if do_backward else None)
        if q2 is not None:
            self._forward(self.q2_network_target, next_state, ws["q2t_next"])
            self._forward(q2, state, ws["q2_out"], ws["q2"] if do_backward else None)
        a = self._critic_args(batch, ws, pins)
        _lib.check(_lib.lib().rb200_crr_critic_head(a, _lib.cur_stream()), "rb200_crr_critic_head")
        if do_backward:
            for net, w in ((self.q1_network, ws["q1"]), (q2, ws["q2"])):
                if net is not None:
                    backward_wgrad(net.arena, w, state, B)
                    net.arena.finish_grads()  # dueling: folded-layer gradient -> true parameters
        return ws["critic_loss"]

    def _critic_args(self, batch: rlt.DiscreteDqnInput, ws, pins: Pins):
        """The critic head's arguments on workspace `ws`, with the draw of the next-state
        exploration noise; `pins` keeps the tensors they point to alive."""
        B, q2 = ws["B"], self.q2_network
        a = _lib.CrrCriticArgsT()
        a.batch, a.num_actions = B, self.num_actions
        a.actor_next = ws["actor_next"].data_ptr()
        a.noise_next = _lib.ptr(self._noise("next", B, pins))
        a.q1_target_next, a.q1 = ws["q1t_next"].data_ptr(), ws["q1_out"].data_ptr()
        a.action = pins(batch.action)
        a.reward = pins(batch.reward.reshape(-1))
        a.reward_boost = pins(self.reward_boosts.reshape(-1)) if self._has_reward_boost else None
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        a.gamma = float(self.gamma)
        a.td_target, a.q1_selected = ws["td_target"].data_ptr(), ws["q1_sel"].data_ptr()
        a.dz_q1 = ws["q1"].dz[-1].data_ptr()
        if q2 is not None:
            a.q2_target_next, a.q2 = ws["q2t_next"].data_ptr(), ws["q2_out"].data_ptr()
            a.q2_selected, a.dz_q2 = ws["q2_sel"].data_ptr(), ws["q2"].dz[-1].data_ptr()
        a.loss_partials = ws["critic_partials"].data_ptr()
        a.loss = ws["critic_loss"].data_ptr()
        a.tile_counter = ws["counter"][0:1].data_ptr()
        return a

    def _actor_step(self, batch: rlt.DiscreteDqnInput, do_backward: bool = True) -> torch.Tensor:
        """Actor losses with the current q1 (and the actor's gradient partials).  Returns the [2]
        device tensor (actor_loss_without_reg, actor_loss)."""
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        state = pins.tensor(batch.state.float_features)
        B = state.shape[0]
        ws = self._workspace(B, pins.device)
        actor = self.actor_network
        self._forward(self.q1_network, state, ws["q1_out"])
        self._forward(actor, state, ws["actor_out"], ws["actor"] if do_backward else None)
        a = self._actor_args(batch, ws, pins, do_backward)
        _lib.check(_lib.lib().rb200_crr_actor_head(a, _lib.cur_stream()), "rb200_crr_actor_head")
        if do_backward:
            backward_wgrad(actor.arena, ws["actor"], state, B)
        return ws["actor_loss"]

    def _actor_args(self, batch: rlt.DiscreteDqnInput, ws, pins: Pins, do_backward: bool = True):
        """The actor head's arguments on workspace `ws`, with the draw of the current-state
        exploration noise; `pins` keeps the tensors they point to alive."""
        B = ws["B"]
        a = _lib.CrrActorArgsT()
        a.batch, a.num_actions = B, self.num_actions
        a.actor_out, a.q1 = ws["actor_out"].data_ptr(), ws["q1_out"].data_ptr()
        a.noise = _lib.ptr(self._noise("cur", B, pins))
        a.action = pins(batch.action)
        if self.entropy_coeff > 0:
            if batch.extras is None or batch.extras.action_probability is None:
                raise TypeError("entropy_coeff > 0 needs the batch's extras.action_probability")
            prob = batch.extras.action_probability
            if self.strict_input_checks:  # the reference's host-syncing assert (:272)
                assert torch.min(prob) > 0, "Logged action probability <= 0"
            a.action_probability = pins(prob.reshape(-1))
        a.inv_beta = 1 / self.beta
        a.max_weight, a.entropy_coeff = float(self.max_weight), float(self.entropy_coeff)
        a.clip_limit = float(self.clip_limit)
        a.action_activation = self.actor_network.arena.acts[-1]
        a.weight = ws["weight"].data_ptr()
        a.dz = ws["actor"].dz[-1].data_ptr() if do_backward else None
        a.loss_partials = ws["actor_partials"].data_ptr()
        a.loss = ws["actor_loss"].data_ptr()
        a.tile_counter = ws["counter"][1:2].data_ptr()
        return a

    def _cpe_step(self, batch: rlt.DiscreteDqnInput) -> torch.Tensor:
        """:358-367: the next-state propensities come from q1_network_target(next_state) as the
        critic step evaluated it, before any update of this batch."""
        return self._calculate_cpes(batch, next_scores=self._ws["q1t_next"],
                                    constant_discount=True)

    def _actor_batch(self, batch_idx: int) -> bool:
        return batch_idx % self.delayed_policy_update == 0

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int):
        """Yields (q1 loss, [q2 loss,] actor loss or None, [reward loss, cpe loss,] soft update)
        -- :290-388."""
        self._check_input(training_batch)
        closs = self._critic_step(training_batch)
        self.log("td_loss", closs[0], prog_bar=True, batch_size=training_batch.batch_size())
        yield self.fused_loss(closs[0])
        if self.q2_network:
            yield self.fused_loss(closs[1])
        if self._actor_batch(batch_idx):
            aloss = self._actor_step(training_batch)
            self.log("actor_loss_without_reg", aloss[0], prog_bar=True,
                     batch_size=training_batch.batch_size())
            self.log("actor_loss", aloss[1], prog_bar=True,
                     batch_size=training_batch.batch_size())
            yield self.fused_loss(aloss[1])
        else:
            yield None
        if self.calc_cpe_in_training:
            cpe = self._cpe_step(training_batch)
            yield self.fused_loss(cpe[0])
            yield self.fused_loss(cpe[1])
        if self.has_real_reporter:
            self.reporter.log(
                logged_actions=torch.argmax(training_batch.action, dim=1, keepdim=True),
                td_loss=closs[0].detach(),
                logged_propensities=training_batch.extras.action_probability,
                logged_rewards=self.boost_rewards(training_batch.reward, training_batch.action))
        yield self.soft_update_result()

    def train_batch(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int = 0,
                    process_group=None):
        """Fast path: the update of train_step_gen and its optimizers with no host
        synchronisation and without _check_input, the Polyak update of each target folded into
        its network's Adam launch.  Returns (critic losses [2], actor losses [2] or None).  With
        `process_group` (data parallel, equal shards per rank) every gradient is averaged over
        the ranks before its Adam step."""
        from .data_parallel import dp_fused_step

        opts = self.optimizers()
        tau = self.tau
        closs = self._critic_step(training_batch)
        i = 0
        dp_fused_step(opts[i], self.q1_network.arena, process_group,
                      target=self.q1_network_target.arena, tau=tau)
        i += 1
        if self.q2_network:
            dp_fused_step(opts[i], self.q2_network.arena, process_group,
                          target=self.q2_network_target.arena, tau=tau)
            i += 1
        aloss = None
        at, asrc = self.actor_network_target.arena, self.actor_network.arena
        if self._actor_batch(batch_idx):
            aloss = self._actor_step(training_batch)
            dp_fused_step(opts[i], asrc, process_group, target=at, tau=tau)
        else:  # no Adam launch to fold it into: the actor target's soft update on its own
            _lib.check(_lib.lib().rb200_soft_update(at.flat.data_ptr(), asrc.flat.data_ptr(), at.n,
                                                    float(tau), float(1.0 - tau),
                                                    _lib.cur_stream()), "rb200_soft_update")
        i += 1
        if self.calc_cpe_in_training:
            self.cpe_losses = self._cpe_step(training_batch)
            dp_fused_step(opts[i], self.reward_network.arena, process_group)
            dp_fused_step(opts[i + 1], self.q_network_cpe.arena, process_group,
                          target=self.q_network_cpe_target.arena, tau=tau)
        self.all_batches_processed += 1
        return closs, aloss

    @torch.no_grad()
    def validation_step(self, batch, batch_idx: int):
        """(eval_actor_loss_without_reg, eval_actor_loss, eval_td_loss) of `batch`, computed
        without gradients and logged under those names -- :390-440.  As in the reference the
        actor losses are None when `batch_idx` is not an actor batch."""
        if isinstance(batch, dict):
            batch = rlt.DiscreteDqnInput.from_dict(batch)
        td_loss = self._critic_step(batch, do_backward=False)[0].clone()
        without_reg = actor_loss = None
        if self._actor_batch(batch_idx):
            al = self._actor_step(batch, do_backward=False).clone()
            without_reg, actor_loss = al[0], al[1]
        n = batch.batch_size()
        self.log("eval_actor_loss_without_reg", without_reg, batch_size=n)
        self.log("eval_actor_loss", actor_loss, batch_size=n)
        self.log("eval_td_loss", td_loss, batch_size=n)
        return without_reg, actor_loss, td_loss

    def net_grads(self, net):
        """Per-parameter gradients of the last fused backward of `net` (inspection / tests)."""
        return param_grads(net.arena, list(net.parameters()))
