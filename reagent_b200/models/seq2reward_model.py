"""Seq2RewardNetwork (reagent/models/seq2reward_model.py): an nn.LSTM over the action sequence
whose every layer starts from h = map_linear(state[0]), c = 0, and the width-1 head
`lstm_linear` on the top hidden state of the last valid step.

The modules are the reference's, built in its order (`rnn`, `lstm_linear`, `map_linear`), so
`state_dict()` keys and the seeded initial weights are its own; the parameters are then views
of one LstmArena.  The forward is one launch of rb200_seq2reward_forward and `plan` the prefix
tree walk of rb200_seq2reward_plan (csrc/rb200_seq2reward.cu); torch's LSTM never runs.
"""
from typing import Optional

import torch
import torch.nn as nn

from .. import _lib
from ..core import types as rlt
from .base import ModelBase
from .world_model import LstmArena, LstmArenaModule


def check_shape(state_dim, action_dim, num_hiddens, num_hidden_layers, multi_steps=1):
    """Raise if the fused kernels do not take this shape (limits: include/reagent_b200.h)."""
    rc = _lib.lib().rb200_seq2reward_check_shape(state_dim, action_dim, num_hiddens,
                                                 num_hidden_layers, multi_steps)
    _lib.check(rc, "Seq2RewardNetwork")


class Seq2RewardBuffers:
    """Device buffers of one [T, B] shape: acc_reward, the target and loss reduction, the step
    labels and (for training) h / c of every step, gate activations, dy, dGates and dh0."""

    def __init__(self, net: "Seq2RewardNetwork", T: int, B: int, multi_steps: int, device,
                 train: bool):
        H, L = net.num_hiddens, net.num_hidden_layers
        e = lambda *s: torch.empty(*s, device=device)  # noqa: E731
        self.T, self.B, self.k, self.device, self.train = T, B, multi_steps, device, train
        self.acc_reward = e(B, 1)
        self.target = e(B)
        self.loss_partials = torch.zeros(-(-B // _lib.SEQ2REWARD_ROWS_PER_BLOCK), device=device)
        self.counter = torch.zeros(1, dtype=torch.int32, device=device)
        self.loss = torch.zeros(1, device=device)
        self.step_labels = e(B, max(multi_steps, 1))
        if train:
            self.hs = e(L, T + 1, B, H)
            self.cs = e(L, T + 1, B, H)
            self.acts = e(L, T, B, 4 * H)
            self.dgates = e(L, T, B, 4 * H)
            self.dy = e(T, B)
            self.dh0 = e(B, H)

    def discount(self, gamma: float) -> torch.Tensor:
        """[T] fp32(gamma ** t), as the reference's gamma_mask (torch.Tensor of Python floats);
        copied to the device once per gamma."""
        if getattr(self, "_gamma", None) != gamma:
            d = torch.tensor([gamma ** i for i in range(self.T)], dtype=torch.float32)
            self._discount, self._gamma = d.to(self.device), gamma
        return self._discount

    def fits(self, T, B, multi_steps, device, train):
        return ((self.T, self.B, self.k, self.device) == (T, B, multi_steps, device)
                and (self.train or not train))


def _cuda(t: torch.Tensor, name: str, shape) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.Rb200Error(f"Seq2RewardNetwork: {name} is a {t.device} tensor; reagent_b200 "
                              "runs on CUDA only (there is no CPU path)")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"Seq2RewardNetwork: {name} has shape {tuple(t.shape)}, expected "
                         f"{tuple(shape)}")
    return t.float().contiguous()


class Seq2RewardNetwork(LstmArenaModule, ModelBase):
    def __init__(self, state_dim, action_dim, num_hiddens, num_hidden_layers) -> None:
        super().__init__()
        self.state_dim = state_dim
        self.action_dim = action_dim
        self.num_hiddens = num_hiddens
        self.num_hidden_layers = num_hidden_layers
        self.rnn = nn.LSTM(input_size=action_dim, hidden_size=num_hiddens,
                           num_layers=num_hidden_layers)
        self.lstm_linear = nn.Linear(num_hiddens, 1)
        self.map_linear = nn.Linear(state_dim, self.num_hiddens)
        self._arena = self._new_arena()
        self._arena.flatten(self.parameters())
        self._plan_ws = {}

    def _new_arena(self):
        return LstmArena(self.action_dim, self.num_hiddens, self.num_hidden_layers, 1,
                         extra=[(self.num_hiddens, self.state_dim), (self.num_hiddens,)])

    def input_prototype(self):
        return (rlt.FeatureData(torch.randn(1, 1, self.state_dim)),
                rlt.FeatureData(torch.randn(1, 1, self.action_dim)))

    def args(self, T: int, B: int, multi_steps: int = 1) -> "_lib.Seq2rewardArgsT":
        """The shape and arena fields of the kernels' arguments for a [T, B] batch."""
        check_shape(self.state_dim, self.action_dim, self.num_hiddens, self.num_hidden_layers,
                    multi_steps)
        a = _lib.Seq2rewardArgsT()
        a.seq_len, a.batch = T, B
        a.state_dim, a.action_dim = self.state_dim, self.action_dim
        a.hidden, a.layers = self.num_hiddens, self.num_hidden_layers
        ar = self._arena
        ar.fill_lstm(a)
        L = self.num_hidden_layers
        a.w_lin_off, a.b_lin_off, a.w_map_off, a.b_map_off = ar.offsets[4 * L: 4 * L + 4]
        return a

    def forward(self, state: rlt.FeatureData, action: rlt.FeatureData,
                valid_reward_len: Optional[torch.Tensor] = None) -> rlt.Seq2RewardOutput:
        """acc_reward [B, 1] of the reference's forward, from one launch.  Only state[0] is
        read, so a state of seq_len 1 (as get_Q passes it) is accepted."""
        ws = run_forward(self, state.float_features, action.float_features, valid_reward_len)
        return rlt.Seq2RewardOutput(acc_reward=ws.acc_reward)

    @torch.no_grad()
    def plan(self, state: torch.Tensor, multi_steps: int, all_horizons: bool = False):
        """get_Q over every action sequence of length `multi_steps`, by the prefix-tree walk:
        q [B, A] (the max over the sequences that start with each action) and, with
        `all_horizons`, q_all [B, multi_steps, A] with the same max for every length 1..k
        (else None).  No host synchronisation."""
        if state.dim() != 2:
            raise ValueError(f"Seq2RewardNetwork.plan: state must be [B, state_dim], got "
                             f"{tuple(state.shape)}")
        B, A, k = state.shape[0], self.action_dim, multi_steps
        state = _cuda(state, "state", (B, self.state_dim))
        _lib.require_current_device(state.device)
        pa = _lib.Seq2rewardPlanArgsT()
        pa.net = self.args(1, B, k)
        lib = _lib.lib()
        nbytes = int(lib.rb200_seq2reward_plan_workspace_bytes(B, A, k, self.num_hiddens,
                                                               self.num_hidden_layers))
        key = (B, k, state.device)
        ws = self._plan_ws.get(key)
        if ws is None:
            self._plan_ws.clear()
            ws = {"qbits": torch.empty(B, k, A, dtype=torch.int32, device=state.device),
                  "workspace": torch.empty(max(nbytes // 4, 1), device=state.device)}
            self._plan_ws[key] = ws
        q = torch.empty(B, A, device=state.device)
        q_all = torch.empty(B, k, A, device=state.device) if all_horizons else None
        pa.batch, pa.multi_steps = B, k
        pa.state, pa.q = state.data_ptr(), q.data_ptr()
        pa.q_all = None if q_all is None else q_all.data_ptr()
        pa.qbits = ws["qbits"].data_ptr()
        pa.workspace, pa.workspace_bytes = ws["workspace"].data_ptr(), nbytes
        _lib.check(lib.rb200_seq2reward_plan(pa, _lib.cur_stream()), "rb200_seq2reward_plan")
        return q, q_all


def run_forward(net: Seq2RewardNetwork, states, actions, valid_step=None,
                ws: Optional[Seq2RewardBuffers] = None, reward=None, gamma: float = 1.0,
                train: bool = False, multi_steps: int = 0) -> Seq2RewardBuffers:
    """One rb200_seq2reward_forward launch on states [T_s, B, S] (only states[0] is read) and
    actions [T, B, A].  `reward` [T, B] adds the target, the MSE (ws.loss) and, with
    `multi_steps`, the one-hot step labels; `train` keeps what the backward reads.  Returns the
    workspace (fresh buffers when none is passed)."""
    if states.dim() != 3 or actions.dim() != 3:
        raise ValueError(f"Seq2RewardNetwork: state and action must be [T, B, dim], got "
                         f"{tuple(states.shape)} and {tuple(actions.shape)}")
    T, B = actions.shape[0], actions.shape[1]
    a = net.args(T, B)
    state0 = _cuda(states[0], "state[0]", (B, net.state_dim))
    actions = _cuda(actions, "action", (T, B, net.action_dim))
    _lib.require_current_device(state0.device)
    keep = [state0, actions]  # alive until the launch is enqueued
    if ws is None:
        ws = Seq2RewardBuffers(net, T, B, multi_steps, state0.device, train)
    a.state, a.action = state0.data_ptr(), actions.data_ptr()
    if valid_step is not None:
        valid_step = valid_step.reshape(-1)
        if valid_step.shape[0] != B or valid_step.device != state0.device:
            raise ValueError(f"Seq2RewardNetwork: valid_step must have {B} entries on "
                             f"{state0.device}, got {tuple(valid_step.shape)} on "
                             f"{valid_step.device}")
        valid_step = valid_step.to(torch.int64).contiguous()
        keep.append(valid_step)
        a.valid_step = valid_step.data_ptr()
    a.acc_reward = ws.acc_reward.data_ptr()
    if reward is not None:
        reward = _cuda(reward, "reward", (T, B))
        discount = ws.discount(gamma)
        keep.append(reward)
        a.reward, a.discount, a.target = reward.data_ptr(), discount.data_ptr(), ws.target.data_ptr()
        a.loss_partials, a.tile_counter = ws.loss_partials.data_ptr(), ws.counter.data_ptr()
        a.loss = ws.loss.data_ptr()
        if multi_steps:
            a.step_labels, a.multi_steps = ws.step_labels.data_ptr(), multi_steps
    if train:
        a.hs, a.cs, a.acts, a.dy = (ws.hs.data_ptr(), ws.cs.data_ptr(), ws.acts.data_ptr(),
                                    ws.dy.data_ptr())
    _lib.check(_lib.lib().rb200_seq2reward_forward(a, _lib.cur_stream()),
               "rb200_seq2reward_forward")
    ws.keep = keep
    return ws


def backward_wgrad(net: Seq2RewardNetwork, ws: Seq2RewardBuffers, splits: int, gpart):
    """rb200_seq2reward_backward and rb200_seq2reward_wgrad after a training forward on `ws`
    (whose `keep` still holds the forward's state and actions)."""
    state0, actions = ws.keep[0], ws.keep[1]
    a = net.args(ws.T, ws.B)
    a.state, a.action = state0.data_ptr(), actions.data_ptr()
    a.hs, a.cs, a.acts, a.dy = ws.hs.data_ptr(), ws.cs.data_ptr(), ws.acts.data_ptr(), ws.dy.data_ptr()
    a.dgates, a.dh0 = ws.dgates.data_ptr(), ws.dh0.data_ptr()
    lib, st = _lib.lib(), _lib.cur_stream()
    _lib.check(lib.rb200_seq2reward_backward(a, st), "rb200_seq2reward_backward")
    a.splits, a.gpart = splits, gpart.data_ptr()
    _lib.check(lib.rb200_seq2reward_wgrad(a, st), "rb200_seq2reward_wgrad")
    net.arena.grad_ready = True
