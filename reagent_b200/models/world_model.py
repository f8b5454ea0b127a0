"""MemoryNetwork and MDNRNN (reagent/models/world_model.py, reagent/models/mdn_rnn.py): an
nn.LSTM over cat(action, state) with the mixture-density head `gmm_linear`.

The modules are the reference's, so `state_dict()` keys, shapes and the seeded initial
weights are its own; every parameter is then re-pointed at a view of ONE flat arena
(`LstmArena`) in `parameters()` order, which FusedAdam updates in one launch.  The forward is
one launch of rb200_mdnrnn_forward (csrc/rb200_mdnrnn.cu); torch's LSTM never runs.
"""
import copy
from typing import Optional

import torch
import torch.nn as nn

from .. import _lib
from ..core import types as rlt
from .arena import ParamArena, _align4
from .base import ModelBase


class LstmArena(ParamArena):
    """Flat layout of an LSTM network: per layer weight_ih, weight_hh, bias_ih, bias_hh, then
    the head's weight and bias (MDNRNN.gmm_linear, Seq2RewardNetwork.lstm_linear), then any
    `extra` shapes (Seq2RewardNetwork.map_linear), each on a 16-byte boundary."""

    def __init__(self, input_dim: int, hidden: int, layers: int, out_dim: int, extra=()):
        self.dims, self.acts, self.w_off, self.b_off = [], [], [], []
        self.input_dim, self.hidden, self.layers, self.out_dim = input_dim, hidden, layers, out_dim
        self.shapes = []
        for l in range(layers):
            k = input_dim if l == 0 else hidden
            self.shapes += [(4 * hidden, k), (4 * hidden, hidden), (4 * hidden,), (4 * hidden,)]
        self.shapes += [(out_dim, hidden), (out_dim,)] + [tuple(e) for e in extra]
        self.offsets = []
        off = 0
        for s in self.shapes:
            self.offsets.append(off)
            n = 1
            for v in s:
                n *= v
            off = _align4(off + n)
        self.n = off
        self.flat = None
        self.gpart = None
        self.grad_ready = False
        self._desc = None

    def flatten(self, params, device=None):
        """Copy `params` (parameters() order) into a fresh flat buffer and re-point their
        `.data` at views of it."""
        params = list(params)
        assert [tuple(p.shape) for p in params] == self.shapes
        dev = device if device is not None else params[0].device
        flat = torch.zeros(self.n, dtype=torch.float32, device=dev)
        for p, off, s in zip(params, self.offsets, self.shapes):
            v = flat[off: off + p.numel()].view(s)
            v.copy_(p.data.to(dev, torch.float32))
            p.data = v
            p._rb200_arena = self
        self.flat = flat
        self.gpart = None
        self.grad_ready = False
        return flat

    def fill_lstm(self, a):
        """The arena pointer and LSTM layer offsets of the kernels' arguments."""
        a.params = self.flat.data_ptr()
        a.n_params = self.n
        for l in range(self.layers):
            a.w_ih_off[l], a.w_hh_off[l], a.b_ih_off[l], a.b_hh_off[l] = self.offsets[4 * l: 4 * l + 4]

    def fill(self, a: "_lib.MdnrnnArgsT"):
        """The arena fields of the MDN-RNN kernels' arguments."""
        self.fill_lstm(a)
        a.w_gmm_off, a.b_gmm_off = self.offsets[4 * self.layers: 4 * self.layers + 2]


def check_shape(state_dim, action_dim, num_hiddens, num_hidden_layers, num_gaussians):
    """Raise if the fused kernels do not take this shape (limits: include/reagent_b200.h)."""
    rc = _lib.lib().rb200_mdnrnn_check_shape(state_dim, action_dim, num_hiddens,
                                             num_hidden_layers, num_gaussians)
    _lib.check(rc, "MDNRNN")


class LstmArenaModule(nn.Module):
    """A module whose parameters live in the LstmArena of `_new_arena()`, kept there across
    `.to()` / `.cuda()` and deep copies."""

    @property
    def arena(self) -> LstmArena:
        return self._arena

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        # parameters were moved one by one (and nn.LSTM may re-pack them for cuDNN): gather
        # them into a fresh flat buffer again
        self._arena.flatten(self.parameters())
        return self

    def __deepcopy__(self, memo):
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k != "_arena":
                new.__dict__[k] = copy.deepcopy(v, memo)
        new._arena = new._new_arena()
        new._arena.flatten(new.parameters())
        return new


class MDNRNN(LstmArenaModule):
    """Mixture Density Network - Recurrent Neural Network"""

    def __init__(self, state_dim, action_dim, num_hiddens, num_hidden_layers, num_gaussians):
        super().__init__()
        self.state_dim = state_dim
        self.action_dim = action_dim
        self.num_hiddens = num_hiddens
        self.num_hidden_layers = num_hidden_layers
        self.rnn = nn.LSTM(input_size=state_dim + action_dim, hidden_size=num_hiddens,
                           num_layers=num_hidden_layers)
        self.num_gaussians = num_gaussians
        # outputs: mu, sigma and pi of every gaussian, then reward and the non-terminal logit
        self.gmm_linear = nn.Linear(num_hiddens, (2 * state_dim + 1) * num_gaussians + 2)
        self._arena = self._new_arena()
        self._arena.flatten(self.parameters())

    def _new_arena(self):
        return LstmArena(self.state_dim + self.action_dim, self.num_hiddens,
                         self.num_hidden_layers, self.gmm_linear.out_features)

    def args(self, T: int, B: int) -> "_lib.MdnrnnArgsT":
        """The shape and arena fields of the kernels' arguments for a [T, B] batch."""
        check_shape(self.state_dim, self.action_dim, self.num_hiddens, self.num_hidden_layers,
                    self.num_gaussians)
        a = _lib.MdnrnnArgsT()
        a.seq_len, a.batch = T, B
        a.state_dim, a.action_dim = self.state_dim, self.action_dim
        a.hidden, a.layers, a.gaussians = self.num_hiddens, self.num_hidden_layers, self.num_gaussians
        self._arena.fill(a)
        return a

    def forward(self, actions: torch.Tensor, states: torch.Tensor, hidden=None):
        """mus, sigmas, logpi, reward, not_terminal, all_steps_hidden and
        (last_step_hidden, last_step_cell) of the reference's MDNRNN.forward, from one launch."""
        if hidden is not None:
            raise NotImplementedError("MDNRNN.forward: an initial hidden state is not supported "
                                      "(the sequence starts from zeros)")
        out = run_forward(self, states, actions)
        return (out.mus, out.sigmas, out.logpi, out.reward, out.not_terminal,
                out.all_steps_lstm_hidden, (out.last_step_lstm_hidden, out.last_step_lstm_cell))


class MdnBuffers:
    """Device buffers of one [T, B] shape: outputs, h / c of every step, and (for training)
    the network input, gate activations, dGates, dL/d(gmm_outs) and the loss reduction."""

    def __init__(self, net: MDNRNN, T: int, B: int, device, train: bool):
        H, L, NG = net.num_hiddens, net.num_hidden_layers, net.gmm_linear.out_features
        e = lambda *s: torch.empty(*s, device=device)  # noqa: E731
        self.T, self.B, self.device, self.train = T, B, device, train
        self.out = e(T, B, NG)
        self.hs = e(L, T + 1, B, H)
        self.cs = e(L, T + 1, B, H)
        n_blocks = -(-B // _lib.MDNRNN_ROWS_PER_BLOCK)
        self.loss_partials = torch.zeros(3 * n_blocks, device=device)
        self.counter = torch.zeros(1, dtype=torch.int32, device=device)
        self.loss = torch.zeros(4, device=device)
        if train:
            self.xin = e(T, B, net.state_dim + net.action_dim)
            self.acts = e(L, T, B, 4 * H)
            self.dgates = e(L, T, B, 4 * H)
            self.dy = e(T, B, NG)

    def fits(self, T, B, device, train):
        return (self.T, self.B, self.device) == (T, B, device) and (self.train or not train)

    def output(self, net: MDNRNN) -> rlt.MemoryNetworkOutput:
        T, B, S, G = self.T, self.B, net.state_dim, net.num_gaussians
        GS = G * S
        o = self.out
        return rlt.MemoryNetworkOutput(
            mus=o[:, :, :GS].reshape(T, B, G, S), sigmas=o[:, :, GS:2 * GS].reshape(T, B, G, S),
            logpi=o[:, :, 2 * GS:2 * GS + G], reward=o[:, :, -2], not_terminal=o[:, :, -1],
            last_step_lstm_hidden=self.hs[:, T], last_step_lstm_cell=self.cs[:, T],
            all_steps_lstm_hidden=self.hs[-1, 1:])


def _seq(t: torch.Tensor, name: str, T=None, B=None, D=None) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.Rb200Error(f"MDNRNN: {name} is a {t.device} tensor; reagent_b200 runs on "
                              "CUDA only (there is no CPU path)")
    want = tuple(v for v in (T, B, D) if v is not None)
    if tuple(t.shape) != want:
        raise ValueError(f"MDNRNN: {name} has shape {tuple(t.shape)}, expected {want}")
    return t.float().contiguous()


def run_forward(net: MDNRNN, states, actions, ws: Optional[MdnBuffers] = None,
                targets=None, train: bool = False, loss_params=None) -> rlt.MemoryNetworkOutput:
    """One rb200_mdnrnn_forward launch.  `targets` = (next_state, reward, not_terminal) adds the
    loss (into ws.loss); `train` also keeps what the backward reads.  Returns views of the
    output buffers of `ws` (of fresh buffers when no workspace is passed)."""
    if states.dim() != 3:
        raise ValueError(f"MDNRNN: states must be [T, B, state_dim], got {tuple(states.shape)}")
    T, B = states.shape[0], states.shape[1]
    a = net.args(T, B)  # refuses unsupported shapes before anything else
    states = _seq(states, "states", T, B, net.state_dim)
    actions = _seq(actions, "actions", T, B, net.action_dim)
    _lib.require_current_device(states.device)
    keep = [states, actions]  # alive until the launch is enqueued
    if ws is None:
        ws = MdnBuffers(net, T, B, states.device, False)
    a.state, a.action = states.data_ptr(), actions.data_ptr()
    a.out, a.hs, a.cs = ws.out.data_ptr(), ws.hs.data_ptr(), ws.cs.data_ptr()
    if targets is not None:
        ns, r, nt = targets
        ns = _seq(ns, "next_state", T, B, net.state_dim)
        r = _seq(r, "reward", T, B)
        nt = _seq(nt, "not_terminal", T, B)
        keep += [ns, r, nt]
        a.next_state, a.reward, a.not_terminal = ns.data_ptr(), r.data_ptr(), nt.data_ptr()
        (a.next_state_weight, a.not_terminal_weight, a.reward_weight, a.gmm_divisor,
         a.fit_only_one_next_step) = loss_params
        a.loss_partials, a.tile_counter = ws.loss_partials.data_ptr(), ws.counter.data_ptr()
        a.loss = ws.loss.data_ptr()
    if train:
        a.xin, a.acts, a.dgates, a.dy = (ws.xin.data_ptr(), ws.acts.data_ptr(),
                                         ws.dgates.data_ptr(), ws.dy.data_ptr())
    _lib.check(_lib.lib().rb200_mdnrnn_forward(a, _lib.cur_stream()), "rb200_mdnrnn_forward")
    return ws.output(net)


class MemoryNetwork(ModelBase):
    def __init__(self, state_dim, action_dim, num_hiddens, num_hidden_layers, num_gaussians) -> None:
        super().__init__()
        self.mdnrnn = MDNRNN(state_dim=state_dim, action_dim=action_dim, num_hiddens=num_hiddens,
                             num_hidden_layers=num_hidden_layers, num_gaussians=num_gaussians)
        self.state_dim = state_dim
        self.action_dim = action_dim
        self.num_hiddens = num_hiddens
        self.num_hidden_layers = num_hidden_layers
        self.num_gaussians = num_gaussians

    def input_prototype(self):
        return (rlt.FeatureData(torch.randn(1, 1, self.state_dim)),
                rlt.FeatureData(torch.randn(1, 1, self.action_dim)))

    @property
    def arena(self) -> LstmArena:
        return self.mdnrnn.arena

    def forward(self, state: rlt.FeatureData, action: rlt.FeatureData) -> rlt.MemoryNetworkOutput:
        return run_forward(self.mdnrnn, state.float_features, action.float_features)
