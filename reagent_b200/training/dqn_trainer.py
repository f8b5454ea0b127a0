"""DQNTrainer with the reference's constructor, optimizer list and generator protocol
(reagent/training/dqn_trainer.py:27-304), computed by three CUDA launches:

  rb200_dqn_td_step   (K2+K2') TD target, loss, dZ chain        dqn_trainer.py:157-239
  rb200_mlp_wgrad     weight gradients (split-K partials)        autograd Linear backward
  rb200_adam_soft_update (K3)  Adam + Polyak                     optimizer.py:64-85, soft_update.py:47-71

With `bcq=BCQConfig(...)` two launches run before K2: the imitator's fused forward on next_state
(rb200_mlp_forward) and rb200_bcq_filter, whose filtered next-action mask K2 reads in place of
the batch's (dqn_trainer.py:206-220).
"""
from dataclasses import dataclass
from typing import List, Optional

import os

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import EvaluationParameters, RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .dqn_trainer_base import DQNTrainerBaseLightning
from .workspace import (NetWorkspace, Pins, batch_device, check_sample_weight, discount_source,
                        param_grads, wgrad, ws_fits)


@dataclass(frozen=True)
class BCQConfig:
    drop_threshold: float = 0.1


class DQNTrainer(DQNTrainerBaseLightning):
    def __init__(
        self,
        q_network,
        q_network_target,
        reward_network=None,
        q_network_cpe=None,
        q_network_cpe_target=None,
        metrics_to_score=None,
        evaluation: Optional[EvaluationParameters] = None,
        imitator=None,
        actions: Optional[List[str]] = None,
        rl: Optional[RLParameters] = None,
        double_q_learning: bool = True,
        bcq: Optional[BCQConfig] = None,
        minibatch_size: int = 1024,
        minibatches_per_step: int = 1,
        optimizer: Optional[Optimizer__Union] = None,
    ) -> None:
        # @resolve_defaults in the reference (dqn_trainer.py:50): default_factory fields
        evaluation = EvaluationParameters() if evaluation is None else evaluation
        actions = [] if actions is None else actions
        rl = RLParameters() if rl is None else rl
        optimizer = Optimizer__Union.default() if optimizer is None else optimizer
        super().__init__(rl, metrics_to_score=metrics_to_score, actions=actions,
                         evaluation_parameters=evaluation)
        assert self._actions is not None, "Discrete-action DQN needs action names"
        self.double_q_learning = double_q_learning
        self.minibatch_size = minibatch_size
        self.minibatches_per_step = minibatches_per_step or 1
        self.q_network = q_network
        self.q_network_target = q_network_target
        self.q_network_optimizer = optimizer
        self._initialize_cpe(reward_network, q_network_cpe, q_network_cpe_target,
                             optimizer=optimizer)
        # Batch constrained q-learning (dqn_trainer.py:112-117): the imitator is a frozen
        # behaviour-policy network; it is in no optimizer and no soft update
        self.bcq = bcq is not None
        if self.bcq:
            self._check_bcq_imitator(imitator)
            self.bcq_drop_threshold = bcq.drop_threshold
            self.bcq_imitator = imitator
        self._ws = None
        self.all_action_scores = None
        self.bcq_next_actions_mask = None  # [B,A] mask the last TD step handed to K2 (BCQ)
        self._kernel_events = None  # bench hook: list collecting (start, end) events of K2

    def _check_bcq_imitator(self, imitator) -> None:
        from ..models.fully_connected_network import FullyConnectedNetwork

        if imitator is None:
            raise ValueError("bcq needs an imitator: the behaviour-policy network whose "
                             "softmax decides which next actions stay possible")
        if not isinstance(imitator, FullyConnectedNetwork):
            raise NotImplementedError(
                "the BCQ imitator must be a reagent_b200.models.FullyConnectedNetwork (its "
                "forward runs on the fused MLP kernel); got " + type(imitator).__name__)
        if imitator.layers[-1] != self.num_actions:
            raise ValueError(f"the BCQ imitator has {imitator.layers[-1]} outputs, but there are "
                             f"{self.num_actions} actions")
        if not self.maxq_learning:
            raise ValueError(
                "bcq needs maxq_learning=True: the imitator filters the max over possible next "
                "actions, and the reference DQNTrainer fails on every batch of BCQ with SARSA "
                "(possible_actions_mask is unbound in train_step_gen)")

    # ------------------------------------------------------------------
    def configure_optimizers(self):
        """[Adam(q_network), (Adam(reward_network), Adam(q_network_cpe) with CPE,)
        SoftUpdate(targets <- sources)] (dqn_trainer.py:119-155)."""
        optimizers = []
        target_params = list(self.q_network_target.parameters())
        source_params = list(self.q_network.parameters())
        optimizers.append(
            self.q_network_optimizer.make_optimizer_scheduler(self.q_network.parameters()))
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
            ntiles = (B + 15) // 16
            ws = {
                "B": B, "dev": device,
                "net": NetWorkspace(self.q_network.arena, B, device),
                "scores": torch.empty(B, self.num_actions, device=device),
                "td_target": torch.empty(B, device=device),
                "q_sel": torch.empty(B, device=device),
                "next_idx": torch.empty(B, dtype=torch.int32, device=device),
                "loss_partials": torch.zeros(ntiles, device=device),
                "loss": torch.zeros(1, device=device),
                "counter": torch.zeros(1, dtype=torch.int32, device=device),
            }
            if self.bcq:
                ws["bcq_logits"] = torch.empty(B, self.num_actions, device=device)
                ws["bcq_mask"] = torch.empty(B, self.num_actions, device=device)
            self._ws = ws
        return self._ws

    def _bcq_filter(self, x: torch.Tensor, mask_in, logits, mask_out) -> torch.Tensor:
        """mask_out = mask_in * (r >= drop_threshold), r = softmax(imitator(x)) / its row max
        (imitator_training.py:12-25): the imitator's fused forward, then rb200_bcq_filter.
        `x` is a contiguous fp32 [B,S] device tensor, `mask_in` a device pointer or None (ones)."""
        im = self.bcq_imitator
        if im.arena.flat.device != mask_out.device:
            raise _lib.Rb200Error(f"DQNTrainer: the BCQ imitator lives on {im.arena.flat.device}, "
                                  f"the batch on {mask_out.device} (call trainer.to(device))")
        im.arena.forward(x, logits)
        rc = _lib.lib().rb200_bcq_filter(logits.data_ptr(), x.shape[0], self.num_actions,
                                         float(self.bcq_drop_threshold), mask_in,
                                         mask_out.data_ptr(), None, None, _lib.cur_stream())
        _lib.check(rc, "rb200_bcq_filter")
        return mask_out

    def _cpe_next_mask(self, batch: rlt.DiscreteDqnInput) -> Optional[torch.Tensor]:
        """The next-action mask the CPE head sees.  The reference filters with
        `possible_next_actions_mask = batch.possible_next_actions_mask.float(); mask *= keep`
        (dqn_trainer.py:206-216): that writes the batch tensor itself exactly when it already is
        float32, and _calculate_cpes then reads the filtered mask.  This trainer never writes
        the batch (the replay buffer hands every batch the same cached mask tensor), so it passes
        the filtered mask explicitly in that case and leaves the batch mask otherwise."""
        m = batch.possible_next_actions_mask
        if self.bcq and self.maxq_learning and m is not None and m.dtype == torch.float32:
            return self.bcq_next_actions_mask
        return None

    _tc_prepacked = False  # set by a caller that already ran rb200_dqn_tc_pack (fused_step.py)

    def _tc_pack(self, qd, a, device):
        """Scratch for the wgmma path of K2 (packed weight images), or None: see _tc_pack_for."""
        return self._tc_pack_for((int(a.double_q), int(a.do_backward)), qd, device)

    def _tc_pack_for(self, key, qd, device):
        """Weight-image scratch of the wgmma K2 (dqn_td_tc_kernel) for `key` = (double_q,
        do_backward), cached per key, or None when the network's shapes do not fit that kernel:
        then K2 runs on the mma.sync row-tile kernel (dqn_td_rows_kernel).  Both are this
        library's CUDA kernels; there is no other fallback.  Setting RB200_DISABLE_WGMMA before
        a key's first step puts K2 on dqn_td_rows_kernel for every shape, so that kernel can be
        checked on the shapes the wgmma kernel takes; nothing else reads it."""
        cache = self.__dict__.setdefault("_tc_pack_cache", {})
        pack = cache.get(key, False)
        if pack is False or (pack is not None and pack.device != device):
            nbytes = 0
            if not os.environ.get("RB200_DISABLE_WGMMA"):
                nbytes = int(_lib.lib().rb200_dqn_tc_workspace_bytes(qd, key[0], key[1]))
            pack = torch.zeros(nbytes, dtype=torch.uint8, device=device) if nbytes > 0 else None
            cache[key] = pack
        return pack

    def _tc_state(self):
        """What the tensor-core weight images were built from: arena identity, the torch version
        counters of every parameter (in-place torch writes such as load_state_dict bump them;
        the parameters are views, so the arena's own counter does not see those) and the
        library's write epoch of both arenas."""
        qa, ta = self.q_network.arena, self.q_network_target.arena
        return (id(qa.flat), qa.flat._version, getattr(qa, "data_epoch", 0),
                tuple(p._version for p in self.q_network.parameters()),
                id(ta.flat), ta.flat._version, getattr(ta, "data_epoch", 0),
                tuple(p._version for p in self.q_network_target.parameters()))

    def invalidate_tc_images(self):
        """Force the next TD step to rebuild the tensor-core weight images.  Needed only after a
        parameter write that torch's version counters do not record (`p.data.copy_()`, a foreign
        kernel writing into the arena); `load_state_dict`, optimizer steps and `p.copy_()` are
        detected through `_tc_state()`."""
        self._tc_images_state = None

    def _tc_images_current(self) -> bool:
        return self.__dict__.get("_tc_images_state") == self._tc_state()

    def _tc_pack_in_adam(self):
        """(pack, do_backward) for FusedAdam.fused_step when the Adam kernel can write the
        images itself: plain MLP arenas only (a dueling head is re-folded after the step)."""
        from ..models.arena import ParamArena

        qa = self.q_network.arena
        if type(qa) is not ParamArena:
            return None
        pack = self._tc_pack_for((int(bool(self.double_q_learning)), 1), qa.desc(), qa.flat.device)
        return None if pack is None else (pack, 1)

    def tc_prepack(self) -> bool:
        """Build the weight images of the wgmma K2 on the CURRENT stream, for the next
        training `_td_step` (which then skips the packing).  The images depend only on the
        parameters, so a caller may run this on a side stream next to the replay sampling
        (fused_step.py).  Returns False when K2 runs on the row-tile kernel instead."""
        self.q_network.arena.refresh()          # derived parameters (dueling head) first
        self.q_network_target.arena.refresh()
        qd, qtd = self.q_network.arena.desc(), self.q_network_target.arena.desc()
        key = (int(bool(self.double_q_learning)), 1)
        pack = self._tc_pack_for(key, qd, self.q_network.arena.flat.device)
        if pack is None:
            return False
        if not self._tc_images_current():  # else: the last Adam step already wrote them
            rc = _lib.lib().rb200_dqn_tc_pack(qd, qtd, key[0], key[1], pack.data_ptr(),
                                              pack.numel(), _lib.cur_stream())
            _lib.check(rc, "rb200_dqn_tc_pack")
            self._tc_images_state = self._tc_state()
        self._tc_prepacked = True
        return True

    def _td_step(self, batch: rlt.DiscreteDqnInput, do_backward: bool = True,
                 sample_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Fused TD target + loss (+ backward).  Returns the device loss scalar (shape []).
        `sample_weight`: [B] fp32 importance weights (loss = mean(w * loss_row), dZ row * w)."""
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        state = pins.tensor(batch.state.float_features)
        next_state = pins.tensor(batch.next_state.float_features)  # the imitator reads it too
        B = state.shape[0]
        ws = self._workspace(B, pins.device)
        a = _lib.DqnArgsT()
        a.batch = B
        a.state, a.next_state = state.data_ptr(), next_state.data_ptr()
        a.action = pins(batch.action)
        a.next_action = pins(batch.next_action)
        a.reward = pins(batch.reward.reshape(-1))
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        a.possible_next_actions_mask = pins(batch.possible_next_actions_mask)
        if self.bcq and self.maxq_learning:  # the SARSA branch ignores BCQ (dqn_trainer.py:221-227)
            self.bcq_next_actions_mask = self._bcq_filter(
                next_state, a.possible_next_actions_mask, ws["bcq_logits"], ws["bcq_mask"])
            a.possible_next_actions_mask = ws["bcq_mask"].data_ptr()
        src = discount_source(self, batch)
        a.discount_src = pins(src)
        a.discount_mode = _lib.DISCOUNT_CONST if src is None else _lib.DISCOUNT_POW
        a.reward_boost = pins(self.reward_boosts.reshape(-1)) if self._has_reward_boost else None
        a.gamma = float(self.gamma)
        a.double_q = int(bool(self.double_q_learning))
        a.maxq = int(bool(self.maxq_learning))
        a.loss_kind = self.q_network_loss_kind
        a.do_backward = int(do_backward)
        a.all_action_scores = ws["scores"].data_ptr()
        a.td_target = ws["td_target"].data_ptr()
        a.q_selected = ws["q_sel"].data_ptr()
        a.next_action_idx = ws["next_idx"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        if sample_weight is not None:
            a.sample_weight = pins(check_sample_weight(sample_weight, B))
        self.q_network.arena.refresh()          # no-op for plain MLPs; folds a dueling head
        self.q_network_target.arena.refresh()
        qd, qtd = self.q_network.arena.desc(), self.q_network_target.arena.desc()
        ev = self._kernel_events
        if ev is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        pack = self._tc_pack(qd, a, state.device)
        if pack is not None:
            rc = _lib.lib().rb200_dqn_td_step_tc(qd, qtd, a, ws["net"].c, pack.data_ptr(),
                                                 pack.numel(),
                                                 int(do_backward and self._tc_images_current()),
                                                 _lib.cur_stream())
            if do_backward:
                self._tc_prepacked = False
                self._tc_images_state = self._tc_state()  # packed by this call if they were not
            _lib.check(rc, "rb200_dqn_td_step_tc")
        else:
            rc = _lib.lib().rb200_dqn_td_step(qd, qtd, a, ws["net"].c, _lib.cur_stream())
            _lib.check(rc, "rb200_dqn_td_step")
        # profiling hook (re-launch)
        self._last_td_call = (qd, qtd, a, ws["net"].c, pins.keep, pack)
        if ev is not None:
            e1.record()
            ev.append((e0, e1))
        if do_backward:
            wgrad(self.q_network.arena, ws["net"], state, B)
            self.q_network.arena.finish_grads()  # dueling: folded-layer gradient -> true parameters
        self.all_action_scores = ws["scores"]
        return ws["loss"].reshape(())

    # ------------------------------------------------------------------
    def train_step_gen(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int):
        """Yields (td_loss, [reward_loss, cpe_metric_loss,] soft_update_loss) --
        dqn_trainer.py:241-304."""
        self._check_input(training_batch)
        td_loss = self._td_step(training_batch)
        yield self.fused_loss(td_loss)
        td_loss = td_loss.detach()
        if self.calc_cpe_in_training:
            # evaluated here, after the q-network's optimizer step, like the reference's
            # generator (dqn_trainer.py:266-279)
            cpe = self._calculate_cpes(training_batch, self._cpe_next_mask(training_batch))
            yield self.fused_loss(cpe[0])
            yield self.fused_loss(cpe[1])
        if self.has_real_reporter or self.logger:
            self._log_dqn(td_loss, training_batch)
        yield self.soft_update_result()

    def train_batch(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int = 0,
                    process_group=None, importance_weights: Optional[torch.Tensor] = None):
        """Fast path: one full update in 3 launches, Polyak fused into the Adam kernel.
        Same arithmetic as driving train_step_gen with reagent_b200.training.loop.
        `importance_weights` ([B] fp32 on the batch's device, prioritized replay): the TD loss
        becomes mean_i(w_i * loss_i) and row i of dZ is scaled by w_i; the CPE losses stay
        unweighted.
        With `process_group` (data parallel, one rank per GPU, equal shards): the flat
        gradient is summed over ranks and scaled by 1/world before Adam (every loss is a batch
        mean, SURVEY.md 8e) -- inside the Adam kernel over NVLink peer memory when
        data_parallel.enable_p2p(group) was called, else by ONE NCCL all-reduce."""
        self._td_step(training_batch, sample_weight=importance_weights)
        tcp = self._tc_pack_in_adam() if self._last_td_call[-1] is not None else None
        if self.adam_step(self.q_network.arena, process_group, tc_pack=tcp):
            self._tc_images_state = self._tc_state()
        if self.calc_cpe_in_training:
            cpe = self._calculate_cpes(training_batch, self._cpe_next_mask(training_batch))
            self.adam_step(self.reward_network.arena, process_group)
            self.adam_step(self.q_network_cpe.arena, process_group)
            self.cpe_losses = cpe
        self.all_batches_processed += 1
        return self._ws["loss"]

    @torch.no_grad()
    def compute_td_loss_only(self, batch: rlt.DiscreteDqnInput) -> torch.Tensor:
        """validation_step's eval_td_loss (dqn_trainer.py:363-379): forward/loss, no grads."""
        return self._td_step(batch, do_backward=False).clone()

    @torch.no_grad()
    def _scores(self, net, state):
        x = state.float_features if isinstance(state, rlt.FeatureData) else state
        x = x.float().contiguous()
        out = torch.empty(x.shape[0], self.num_actions, device=x.device)
        net.arena.refresh()
        net.arena.forward(x, out)
        return out

    def get_detached_model_outputs(self, state):
        """(q_network(s), q_network_target(s)) on the fused MLP forward (dqn_trainer.py:158-164)."""
        return self._scores(self.q_network, state), self._scores(self.q_network_target, state)

    def page_model_outputs(self, state):
        """q_network(s) alone: the page does not read the target's scores."""
        return self._scores(self.q_network, state)

    def validation_step(self, batch, batch_idx):
        """Log eval_td_loss and return the batch's EvaluationDataPage (dqn_trainer.py:362-379,
        dqn_trainer_base.py:488-496), kept on the batch's device."""
        from ..evaluation.evaluation_data_page import EvaluationDataPage

        if isinstance(batch, dict):
            batch = rlt.DiscreteDqnInput.from_dict(batch)
        self.log("eval_td_loss", self.compute_td_loss_only(batch), batch_size=batch.batch_size())
        return EvaluationDataPage.create_from_training_batch(batch, self)

    def q_network_grads(self):
        """Per-parameter gradients of the last fused backward (inspection / tests)."""
        return param_grads(self.q_network.arena, list(self.q_network.parameters()))

    # ------------------------------------------------------------------
    def _log_dqn(self, td_loss, training_batch):
        """dqn_trainer.py:292-347 -- only evaluated when a reporter/logger is attached."""
        scores = self.all_action_scores
        logged_action_idxs = torch.argmax(training_batch.action, dim=1, keepdim=True)
        rewards = self.boost_rewards(training_batch.reward, training_batch.action)
        mask = (training_batch.possible_actions_mask if self.maxq_learning
                else training_batch.action)
        if self.bcq and self.maxq_learning:  # dqn_trainer.py:287-291, without writing the batch
            pins = Pins(training_batch.state.float_features.device)
            mask = self._bcq_filter(pins.tensor(training_batch.state.float_features), pins(mask),
                                    torch.empty_like(scores), torch.empty_like(scores))
        model_action_idxs = self.get_max_q_values(scores, mask.float())[1]
        extras = training_batch.extras
        self.reporter.log(
            td_loss=td_loss,
            logged_actions=logged_action_idxs,
            logged_propensities=None if extras is None else extras.action_probability,
            logged_rewards=rewards,
            logged_values=None,
            model_values=scores,
            model_values_on_logged_actions=None,
            model_action_idxs=model_action_idxs,
        )
        if self.logger:
            self.logger.log_metrics(
                {"td_loss": td_loss, "logged_rewards": rewards.mean()},
                step=self.all_batches_processed)
