"""C51Trainer (reagent/training/c51_trainer.py:20-214): categorical distributional DQN.  The
distributional network (trunk + wide [hidden -> A*N] head) runs on the same launches as the
QR-DQN path; rb200_c51_head does the log-softmax, masked arg max, categorical projection,
cross-entropy loss and d loss / d logits, one CTA per batch row."""
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import RLParameters
from ..optimizer import Optimizer__Union, SoftUpdate
from .reagent_lightning_module import ReAgentLightningModule
from .rl_trainer_pytorch import RLTrainerMixin
from .workspace import (NetWorkspace, check_sample_weight, head_backward_dx, param_grads,
                        wgrad)


def _f32c(t):
    return None if t is None else t.float().contiguous()


class C51Trainer(RLTrainerMixin, ReAgentLightningModule):
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
        boosts = torch.zeros([1, len(self._actions)])
        self._has_reward_boost = False
        if self.rl_parameters.reward_boost is not None:
            for k in self.rl_parameters.reward_boost.keys():
                boosts[0, self._actions.index(k)] = self.rl_parameters.reward_boost[k]
                self._has_reward_boost = True
        self.register_buffer("reward_boosts", boosts)
        self._ws = None

    @property
    def num_actions(self) -> int:
        return len(self._actions)

    def configure_optimizers(self):
        return [self.q_network_optimizer.make_optimizer_scheduler(self.q_network.parameters()),
                SoftUpdate.make_optimizer_scheduler(list(self.q_network_target.parameters()),
                                                    list(self.q_network.parameters()), tau=self.tau)]

    def _workspace(self, B, device):
        ws = self._ws
        if ws is None or ws["B"] != B or ws["dev"] != device:
            arena = self.q_network.arena
            AN = arena.dims[-1]
            ws = {"B": B, "dev": device, "net": NetWorkspace(arena, B, device),
                  "l_next_online": torch.empty(B, AN, device=device),
                  "l_next_target": torch.empty(B, AN, device=device),
                  "l_cur": torch.empty(B, AN, device=device),
                  "trunk_tmp": (torch.empty(B, arena.dims[-2], device=device)
                                if len(arena.acts) > 1 else None),
                  "all_q": torch.empty(B, self.num_actions, device=device),
                  "next_idx": torch.empty(B, dtype=torch.int32, device=device),
                  "loss_partials": torch.zeros(B, device=device),
                  "loss": torch.zeros(1, device=device),
                  "counter": torch.zeros(1, dtype=torch.int32, device=device)}
            self._ws = ws
        return ws

    def _forward(self, arena, x, out, ws, save):
        """out[B, A*N] = distributional_network(x): fused trunk + 2-D tiled head."""
        lib, st = _lib.lib(), _lib.cur_stream()
        B, L = x.shape[0], len(arena.acts)
        h = x
        if L > 1:
            h = ws["net"].hidden[L - 2] if save else ws["trunk_tmp"]
            rc = lib.rb200_mlp_forward(arena.desc(L - 1), x.data_ptr(), x.shape[1], None, 0, B,
                                       h.data_ptr(), ws["net"].c if save else None, st)
            _lib.check(rc, "rb200_mlp_forward(trunk)")
        f = arena.flat.data_ptr()
        rc = lib.rb200_linear_forward(f + 4 * arena.w_off[L - 1], f + 4 * arena.b_off[L - 1],
                                      arena.acts[L - 1], arena.dims[L - 1], arena.dims[L],
                                      h.data_ptr(), B, out.data_ptr(), st)
        _lib.check(rc, "rb200_linear_forward(head)")

    def _c51_step(self, batch: rlt.DiscreteDqnInput,
                  sample_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`sample_weight`: [B] fp32 importance weights (loss = mean(w * loss_row), dz_logits row
        scaled by w; ws["loss_partials"] keeps the unweighted row cross entropies)."""
        state = _f32c(batch.state.float_features)
        if not state.is_cuda:
            raise _lib.Rb200Error("C51Trainer: training batch must be on the GPU (no CPU path)")
        next_state = _f32c(batch.next_state.float_features)
        dev, B = state.device, state.shape[0]
        _lib.require_current_device(dev)
        ws = self._workspace(B, dev)
        qa, ta = self.q_network.arena, self.q_network_target.arena
        L = len(qa.acts)
        assert qa.dims[-1] == self.num_actions * self.num_atoms
        lib, st = _lib.lib(), _lib.cur_stream()
        dq = self.double_q_learning and self.maxq_learning
        if dq:
            self._forward(qa, next_state, ws["l_next_online"], ws, save=False)
        self._forward(ta, next_state, ws["l_next_target"], ws, save=False)
        self._forward(qa, state, ws["l_cur"], ws, save=True)
        keep = []

        def P(t):
            t = _lib.on_device(_f32c(t), dev)
            keep.append(t)
            return _lib.ptr(t, dev)

        a = _lib.C51ArgsT()
        a.batch, a.num_actions, a.num_atoms = B, self.num_actions, self.num_atoms
        a.logits_next_online = ws["l_next_online"].data_ptr() if dq else None
        a.logits_next_target = ws["l_next_target"].data_ptr()
        a.logits_cur = ws["l_cur"].data_ptr()
        a.action = P(batch.action)
        a.next_action = P(batch.next_action)
        a.possible_next_actions_mask = P(batch.possible_next_actions_mask)
        a.reward = P(batch.reward.reshape(-1))
        a.not_terminal = P(batch.not_terminal.reshape(-1))
        if self.use_seq_num_diff_as_time_diff:
            assert self.multi_steps is None
            a.discount_src = P(batch.time_diff.reshape(-1))
        if self.multi_steps is not None:
            assert batch.step is not None
            a.discount_src = P(batch.step.reshape(-1))
        a.reward_boost = P(self.reward_boosts.reshape(-1)) if self._has_reward_boost else None
        a.support = P(self.support)
        a.gamma, a.qmin, a.qmax = float(self.gamma), float(self.qmin), float(self.qmax)
        a.scale_support = float(self.scale_support)
        a.double_q, a.maxq = int(bool(self.double_q_learning)), int(bool(self.maxq_learning))
        a.dz_logits = ws["net"].dz[L - 1].data_ptr()
        a.all_q_values = ws["all_q"].data_ptr()
        a.next_action_idx = ws["next_idx"].data_ptr()
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.loss = ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        a.sample_weight = P(check_sample_weight(sample_weight, B))
        _lib.check(lib.rb200_c51_head(a, st), "rb200_c51_head")
        if L > 1:
            head_backward_dx(qa, ws["net"], B, ws)
            if L > 2:
                rc = lib.rb200_mlp_backward(qa.desc(L - 1), ws["net"].dz[L - 2].data_ptr(), B, ws["net"].c, st)
                _lib.check(rc, "rb200_mlp_backward")
        wgrad(qa, ws["net"], state, B)
        self.all_q_values = ws["all_q"]
        return ws["loss"].reshape(())

    def train_step_gen(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int):
        loss = self._c51_step(training_batch)
        yield self.fused_loss(loss)
        yield self.soft_update_result()

    def train_batch(self, training_batch: rlt.DiscreteDqnInput, batch_idx: int = 0, process_group=None,
                    importance_weights: Optional[torch.Tensor] = None):
        """`importance_weights` ([B] fp32 on the batch's device, prioritized replay): the loss
        becomes mean_b(w_b * loss_b) over the per-row cross entropies and row b of d loss /
        d logits is scaled by w_b."""
        from .data_parallel import dp_fused_step

        opts = self.optimizers()
        self._c51_step(training_batch, sample_weight=importance_weights)
        dp_fused_step(opts[0], self.q_network.arena, process_group,
                      target=self.q_network_target.arena, tau=self.tau)
        self.all_batches_processed += 1
        return self._ws["loss"]

    @torch.no_grad()
    def boost_rewards(self, rewards: torch.Tensor, actions: torch.Tensor) -> torch.Tensor:
        return rewards + torch.sum(actions.float() * self.reward_boosts, dim=1, keepdim=True)

    def argmax_with_mask(self, q_values, possible_actions_mask):
        q_values = q_values.reshape(possible_actions_mask.shape)
        return (q_values + (-1e9) * (1 - possible_actions_mask)).argmax(1)

    def q_network_grads(self):
        return param_grads(self.q_network.arena, list(self.q_network.parameters()))
