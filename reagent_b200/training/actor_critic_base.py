"""Shared machinery of the fused SAC / TD3 trainers: argument marshalling for
rb200_ac_critic_step / rb200_ac_actor_step, workspaces, noise, weight gradients."""
from typing import Optional

import torch

from .. import _lib
from ..core import types as rlt
from .reagent_lightning_module import ReAgentLightningModule
from .rl_trainer_pytorch import RLTrainerMixin
from .workspace import (NetWorkspace, Pins, batch_device, check_sample_weight, param_grads,
                        wgrad, ws_fits)


class ActorCriticBase(RLTrainerMixin, ReAgentLightningModule):
    ALGO = None

    def _ac_init(self):
        self._ws = None
        # noise_hook(name, shape, device) -> tensor lets tests inject the reference's
        # torch.randn_like draws; default: torch.randn on the device
        self.noise_hook = None
        # (row0, B_global) while a data-parallel step trains rows [row0, row0 + B) of a global
        # batch: the noise is then drawn for the whole batch and the shard takes its rows
        self.noise_rows = None
        self._kernel_events = None

    def _noise(self, name, B, A, pins):
        """Device pointer of a [B, A] standard normal draw (kept alive in `pins`)."""
        if self.noise_hook is not None:
            return pins(self.noise_hook(name, (B, A), pins.device))
        rows = getattr(self, "noise_rows", None)
        if rows is not None:
            row0, batch_global = rows
            return pins(torch.randn(batch_global, A, device=pins.device)[row0:row0 + B])
        return pins(torch.randn(B, A, device=pins.device))

    def _workspace(self, B, device):
        if not ws_fits(self._ws, B, device):
            ntiles = (B + 15) // 16
            q2 = self.q2_network
            value = getattr(self, "value_network", None)
            ws = {
                "B": B, "dev": device,
                "actor": NetWorkspace(self.actor_network.arena, B, device),
                "q1": NetWorkspace(self.q1_network.arena, B, device, need_input=True),
                "q2": None if q2 is None else NetWorkspace(q2.arena, B, device),
                "loss_partials": torch.zeros(2 * ntiles, device=device),
                "critic_loss": torch.zeros(2, device=device),
                "actor_loss": torch.zeros(2, device=device),
                "counter": torch.zeros(1, dtype=torch.int32, device=device),
                "alpha_grad": torch.zeros(1, 1, device=device),
                "td_target": torch.empty(B, device=device),
                "q1_value": torch.empty(B, device=device),
                "q2_value": torch.empty(B, device=device),
                "log_prob": torch.empty(B, device=device),
                # weighted critic step (prioritized replay): max_c |q_c(s, a) - td_target|
                "td_error": torch.empty(B, device=device),
                # SAC with a value network: min_c q_c(s, pi(s)) from the actor step, V's loss
                "value": None if value is None else NetWorkspace(value.arena, B, device),
                "min_q": torch.empty(B, device=device),
                "value_loss": torch.zeros(1, device=device),
            }
            if ws["q2"] is not None:
                ws["q2"].c.input = ws["q1"].input.data_ptr()
            self._ws = ws
        return self._ws

    def _base_args(self, batch: rlt.PolicyNetworkInput, ws, pins):
        """(args, state): the fields both fused steps read, `state` as the fp32 tensor handed
        to them."""
        a = _lib.AcArgsT()
        state = pins.tensor(batch.state.float_features)
        a.batch = state.shape[0]
        a.algo = self.ALGO
        a.state = state.data_ptr()
        a.action = pins(batch.action.float_features)
        a.next_state = pins(batch.next_state.float_features)
        a.reward = pins(batch.reward.reshape(-1))
        a.not_terminal = pins(batch.not_terminal.reshape(-1))
        a.gamma = float(self.gamma)
        a.loss_partials = ws["loss_partials"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        return a, state

    def _desc(self, net):
        return None if net is None else net.arena.desc()

    def _critic_step(self, batch, actor_net, q1t, q2t, fill,
                     sample_weight: Optional[torch.Tensor] = None):
        """`sample_weight`: [B] fp32 importance weights of prioritized replay.  Each critic's
        loss becomes mean(w * (q - y)^2) and row b of its dZ is scaled by w_b; the row's TD
        error max_c |q_c - y| goes to the workspace's "td_error"."""
        B = batch.state.float_features.shape[0]
        check_sample_weight(sample_weight, B)
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        ws = self._workspace(B, pins.device)
        a, _ = self._base_args(batch, ws, pins)
        if sample_weight is not None:
            a.sample_weight = pins(sample_weight)
            a.td_error_out = ws["td_error"].data_ptr()
        if getattr(self, "value_network", None) is None:
            # with a value network the target is V'(s'): no actor forward on s', no draw
            A = self.q1_network.arena.dims[0] - self.actor_network.arena.dims[0]
            a.noise_next = self._noise("next", B, A, pins)
        a.loss = ws["critic_loss"].data_ptr()
        a.td_target = ws["td_target"].data_ptr()
        a.q1_value = ws["q1_value"].data_ptr()
        a.q2_value = ws["q2_value"].data_ptr()
        a.log_prob_out = ws["log_prob"].data_ptr()
        fill(a, pins)
        q2 = self.q2_network
        ev = self._kernel_events
        if ev is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        rc = _lib.lib().rb200_ac_critic_step(
            self._desc(actor_net), self._desc(self.q1_network), self._desc(q2),
            self._desc(q1t), self._desc(q2t), a, ws["q1"].c,
            None if q2 is None else ws["q2"].c, _lib.cur_stream())
        _lib.check(rc, "rb200_ac_critic_step")
        if ev is not None:
            e1.record()
            ev.append((e0, e1))
        wgrad(self.q1_network.arena, ws["q1"], None, B)
        if q2 is not None:
            wgrad(q2.arena, ws["q2"], None, B)
        return ws["critic_loss"]

    def _actor_step(self, batch, fill):
        B = batch.state.float_features.shape[0]
        pins = Pins(batch_device(batch.state.float_features, type(self).__name__))
        ws = self._workspace(B, pins.device)
        a, state = self._base_args(batch, ws, pins)
        a.loss = ws["actor_loss"].data_ptr()
        a.log_prob_out = ws["log_prob"].data_ptr()
        fill(a, pins)
        q2 = self.q2_network
        rc = _lib.lib().rb200_ac_actor_step(
            self._desc(self.actor_network), self._desc(self.q1_network), self._desc(q2), a,
            ws["actor"].c, ws["q1"].c, None if q2 is None else ws["q2"].c, _lib.cur_stream())
        _lib.check(rc, "rb200_ac_actor_step")
        wgrad(self.actor_network.arena, ws["actor"], state, B)
        return ws["actor_loss"]

    def net_grads(self, net):
        """Per-parameter gradients of the last fused backward of `net` (tests)."""
        return param_grads(net.arena, list(net.parameters()))
