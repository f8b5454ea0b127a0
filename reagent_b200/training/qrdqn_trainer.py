"""QRDQNTrainer with the reference's constructor, optimizer list and generator protocol
(reagent/training/qrdqn_trainer.py:21-227, CPE off).

Launches of one update (network [S -> hidden... -> A*N]):
  trunk (fused MLP rows kernel) + wide head (2-D tiled) forward x3   q(s'), q_target(s'), q(s)
  rb200_qrdqn_head        mean over atoms, masked argmax, target distribution,
                          pairwise quantile-Huber loss + d loss/d head output   :125-155
  rb200_linear_backward_dx (head), rb200_mlp_backward (trunk dZ chain)
  rb200_mlp_wgrad, rb200_adam_soft_update
The (N, B, N) pairwise tensor of the reference (655 MB at config 3) is never materialised.
"""
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import EvaluationParameters, RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .dqn_trainer import _f32c
from .dqn_trainer_base import DQNTrainerBaseLightning
from .workspace import (NetWorkspace, check_sample_weight, head_backward_dx, param_grads,
                        wgrad)


class QRDQNTrainer(DQNTrainerBaseLightning):
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
    def _workspace(self, B, device):
        ws = self._ws
        if ws is None or ws["B"] != B or ws["dev"] != device:
            arena = self.q_network.arena
            AN = arena.dims[-1]
            ws = {
                "B": B, "dev": device,
                "net": NetWorkspace(arena, B, device),
                "q_next_online": torch.empty(B, AN, device=device),
                "q_next_target": torch.empty(B, AN, device=device),
                "q_cur": torch.empty(B, AN, device=device),
                "trunk_tmp": (torch.empty(B, arena.dims[-2], device=device)
                              if len(arena.acts) > 1 else None),
                "all_q": torch.empty(B, self.num_actions, device=device),
                "next_idx": torch.empty(B, dtype=torch.int32, device=device),
                "loss_partials": torch.zeros(B, device=device),
                "loss": torch.zeros(1, device=device),
                "counter": torch.zeros(1, dtype=torch.int32, device=device),
            }
            self._ws = ws
        return ws

    def _forward(self, arena, x, out, ws, save):
        """out[B, A*N] = net(x): fused trunk + 2-D tiled head."""
        lib = _lib.lib()
        B = x.shape[0]
        L = len(arena.acts)
        st = _lib.cur_stream()
        h = x
        if L > 1:
            h = ws["net"].hidden[L - 2] if save else ws["trunk_tmp"]
            rc = lib.rb200_mlp_forward(arena.desc(L - 1), x.data_ptr(), x.shape[1], None, 0, B,
                                       h.data_ptr(), ws["net"].c if save else None, st)
            _lib.check(rc, "rb200_mlp_forward(trunk)")
        flat = arena.flat
        rc = lib.rb200_linear_forward(
            flat.data_ptr() + 4 * arena.w_off[L - 1], flat.data_ptr() + 4 * arena.b_off[L - 1],
            arena.acts[L - 1], arena.dims[L - 1], arena.dims[L], h.data_ptr(), B,
            out.data_ptr(), st)
        _lib.check(rc, "rb200_linear_forward(head)")

    def _qr_step(self, batch: rlt.DiscreteDqnInput,
                 sample_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`sample_weight`: [B] fp32 importance weights (loss = mean(w * loss_row), dz_head row
        scaled by w; ws["loss_partials"] keeps the unweighted row sums)."""
        state = _f32c(batch.state.float_features)
        if not state.is_cuda:
            raise _lib.Rb200Error("QRDQNTrainer: training batch must be on the GPU (no CPU path)")
        _lib.require_current_device(state.device)
        next_state = _f32c(batch.next_state.float_features)
        B = state.shape[0]
        ws = self._workspace(B, state.device)
        qa, ta = self.q_network.arena, self.q_network_target.arena
        L = len(qa.acts)
        if qa.dims[-1] != self.num_actions * self.num_atoms:
            raise ValueError("q_network output width must be num_actions * num_atoms")
        lib, st = _lib.lib(), _lib.cur_stream()
        qa.refresh()  # no-op for plain MLPs; folds a dueling head into its last Linear
        ta.refresh()
        if self.double_q_learning and self.maxq_learning:
            self._forward(qa, next_state, ws["q_next_online"], ws, save=False)
        self._forward(ta, next_state, ws["q_next_target"], ws, save=False)
        self._forward(qa, state, ws["q_cur"], ws, save=True)
        keep = []

        def P(t):
            t = _lib.on_device(_f32c(t), state.device)
            keep.append(t)
            return _lib.ptr(t, state.device)

        a = _lib.QrdqnArgsT()
        a.batch, a.num_actions, a.num_atoms = B, self.num_actions, self.num_atoms
        a.q_next_online = ws["q_next_online"].data_ptr()
        a.q_next_target = ws["q_next_target"].data_ptr()
        a.q_cur = ws["q_cur"].data_ptr()
        a.action = P(batch.action)
        a.next_action = P(batch.next_action)
        a.possible_next_actions_mask = P(batch.possible_next_actions_mask)
        a.reward = P(batch.reward.reshape(-1))
        a.not_terminal = P(batch.not_terminal.reshape(-1))
        a.discount_src = None
        if self.use_seq_num_diff_as_time_diff:
            assert self.multi_steps is None
            a.discount_src = P(batch.time_diff.reshape(-1))
        if self.multi_steps is not None:
            assert batch.step is not None
            a.discount_src = P(batch.step.reshape(-1))
        a.reward_boost = P(self.reward_boosts.reshape(-1)) if self._has_reward_boost else None
        a.gamma = float(self.gamma)
        a.double_q = int(bool(self.double_q_learning))
        a.maxq = int(bool(self.maxq_learning))
        a.dz_head = ws["net"].dz[L - 1].data_ptr()
        a.all_q_values = ws["all_q"].data_ptr()
        a.next_action_idx = ws["next_idx"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        a.sample_weight = P(check_sample_weight(sample_weight, B))
        _lib.check(lib.rb200_qrdqn_head(a, st), "rb200_qrdqn_head")
        if L > 1:
            head_backward_dx(qa, ws["net"], B, ws)
            if L > 2:
                rc = lib.rb200_mlp_backward(qa.desc(L - 1), ws["net"].dz[L - 2].data_ptr(), B,
                                            ws["net"].c, st)
                _lib.check(rc, "rb200_mlp_backward")
        wgrad(qa, ws["net"], state, B)
        qa.finish_grads()  # dueling: folded-layer gradient -> true parameters
        self.all_q_values = ws["all_q"]
        return ws["loss"].reshape(())

    def train_step_gen(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int):
        self._check_input(training_batch)
        loss = self._qr_step(training_batch)
        yield self.fused_loss(loss)
        self.loss = loss.detach()
        if self.has_real_reporter:
            logged_action_idxs = torch.argmax(training_batch.action, dim=1, keepdim=True)
            self.reporter.log(
                td_loss=self.loss, logged_actions=logged_action_idxs,
                logged_rewards=self.boost_rewards(training_batch.reward, training_batch.action),
                model_values=self.all_q_values)
        yield self.soft_update_result()

    def train_batch(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int = 0,
                    process_group=None, importance_weights: Optional[torch.Tensor] = None):
        """`importance_weights` ([B] fp32 on the batch's device, prioritized replay): the loss
        becomes mean_b(w_b * loss_b) over the per-row quantile-Huber losses and row b of the
        head gradient is scaled by w_b."""
        opts = self.optimizers()
        self._qr_step(training_batch, sample_weight=importance_weights)
        from .data_parallel import dp_fused_step

        dp_fused_step(opts[0], self.q_network.arena, process_group,
                      target=self.q_network_target.arena, tau=self.tau)
        self.all_batches_processed += 1
        return self._ws["loss"]

    def q_network_grads(self):
        return param_grads(self.q_network.arena, list(self.q_network.parameters()))
