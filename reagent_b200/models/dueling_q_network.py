"""DuelingQNetwork (reagent/models/dueling_q_network.py:20-125) on the fused MLP kernels.

Same constructor, `make_fully_connected` and sub-module names as the reference
(`shared_network`, `advantage_network`, `value_network`, each a FullyConnectedDQN, so
`state_dict()` keys match and reference checkpoints load).  All parameters live in ONE flat
arena; the network is presented to the kernels as the plain MLP it is algebraically equal to:

    [S] -> shared trunk -> E (linear) -> [adv hidden | value hidden] (2H = E) -> A (* atoms)
                                          stacked first head layers        folded last layer

* the first Linear of the two heads are consecutive row blocks of one [E x E] weight (views);
* the last layer W_q / b_q is DERIVED from (W_adv, b_adv, w_val, b_val) by rb200_dueling_fold
  before every use (`arena.refresh()`), and its gradient is mapped back onto the true parameters
  by rb200_dueling_unfold after the weight-gradient kernel (`arena.finish_grads()`).  The
  derived region sits at the end of the arena; Adam / Polyak sweep it too but its gradient is
  zero by then, so it does not move (and it is rebuilt anyway).
The dense heads of `make_fully_connected` are supported, with or without atoms (QR-DQN's
DuelingQuantile: value head N outputs, advantage head A*N, mean over actions AND atoms);
batch norm and the parametric variant raise NotImplementedError.
"""
import copy
from typing import List, Optional

import torch

from .. import _lib
from ..core import types as rlt
from .arena import ParamArena, _align4, run_mlp
from .base import ModelBase, require_cuda
from .dqn import FullyConnectedDQN

INVALID_ACTION_CONSTANT = -1e10


class DuelingArena(ParamArena):
    """Flat layout [shared layers | W_stack, b_stack | W_adv2, b_adv2, w_val2, b_val2 | W_q, b_q]
    described to the kernels as the equivalent plain MLP."""

    def __init__(self, shared_dims: List[int], shared_acts: List[int], head_act: int, A: int,
                 N: int = 1):
        E = shared_dims[-1]
        H = E // 2
        self.E, self.H, self.A, self.N = E, H, A, N
        R = A * N  # output rows of the folded layer: r = a * N + n
        self.dims = list(shared_dims) + [2 * H, R]
        self.acts = list(shared_acts) + [head_act, _lib.ACT["linear"]]
        assert len(self.acts) <= _lib.MAX_LAYERS, f"at most {_lib.MAX_LAYERS} layers are supported"
        self.w_off, self.b_off = [], []
        off = 0
        for i in range(len(shared_acts) + 1):          # shared layers, then the stacked head layer
            self.w_off.append(off)
            off = _align4(off + self.dims[i] * self.dims[i + 1])
            self.b_off.append(off)
            off = _align4(off + self.dims[i + 1])
        self.o_wa, off = off, _align4(off + R * H)      # true parameters of the last head layers
        self.o_ba, off = off, _align4(off + R)
        self.o_wv, off = off, _align4(off + N * H)
        self.o_bv, off = off, _align4(off + N)
        self.n_true = off
        self.w_off.append(off)                          # derived last layer of the plain MLP
        off = _align4(off + R * 2 * H)
        self.b_off.append(off)
        off = _align4(off + R)
        self.n = off
        self.flat: Optional[torch.Tensor] = None
        self.gpart = None
        self.grad_ready = False
        self._scratch = None

    def _scratch_for(self, splits: int):
        need = int(_lib.lib().rb200_dueling_scratch_floats(self.H, splits))
        sc = self._scratch
        if sc is None or sc.numel() < need or sc.device != self.flat.device:
            sc = self._scratch = torch.zeros(need, dtype=torch.float32, device=self.flat.device)
        return sc

    def refresh(self):
        p = self.flat.data_ptr()
        W, b = self.layer_ptrs(len(self.acts) - 1)
        rc = _lib.lib().rb200_dueling_fold(p + 4 * self.o_wa, p + 4 * self.o_ba, p + 4 * self.o_wv,
                                           p + 4 * self.o_bv, self.A, self.N, self.H, W, b,
                                           self._scratch_for(1).data_ptr(), _lib.cur_stream())
        _lib.check(rc, "rb200_dueling_fold")

    def finish_grads(self):
        g = self.gpart
        L = len(self.acts)
        rc = _lib.lib().rb200_dueling_unfold(g.data_ptr(), self.n, g.shape[0], self.A, self.N,
                                             self.H, self.w_off[L - 1], self.b_off[L - 1],
                                             self.o_wa, self.o_ba, self.o_wv, self.o_bv,
                                             self._scratch_for(g.shape[0]).data_ptr(),
                                             _lib.cur_stream())
        _lib.check(rc, "rb200_dueling_unfold")


class DuelingQNetwork(ModelBase):
    def __init__(self, *, shared_network: ModelBase, advantage_network: ModelBase,
                 value_network: ModelBase) -> None:
        super().__init__()
        for name, net in (("shared_network", shared_network),
                          ("advantage_network", advantage_network),
                          ("value_network", value_network)):
            if not isinstance(net, FullyConnectedDQN):
                raise NotImplementedError(
                    f"DuelingQNetwork: {name} must be a FullyConnectedDQN (the "
                    "make_fully_connected structure); other heads are out of scope")
        self.shared_network = shared_network
        self.advantage_network = advantage_network
        self.value_network = value_network
        E = shared_network.output_dim
        adv, val = advantage_network.fc, value_network.fc
        self.num_atoms = advantage_network.num_atoms
        N = self.num_atoms or 1
        ok = (len(adv.layers) == 3 and len(val.layers) == 3 and adv.layers[0] == E
              and val.layers[0] == E and adv.layers[1] == val.layers[1] == E // 2
              and val.layers[2] == N and adv.layers[2] % N == 0
              and value_network.num_atoms == self.num_atoms and shared_network.num_atoms is None
              and adv.activations == val.activations
              and adv.activations[-1] == "linear" and shared_network.fc.activations[-1] == "linear")
        if not ok:
            raise NotImplementedError(
                "DuelingQNetwork: only the make_fully_connected head structure "
                "([E -> E/2 -> A(*N)] and [E -> E/2 -> 1(*N)], linear outputs) is supported")
        self.action_dim = adv.layers[2] // N
        self._name = "unnamed"
        self._build_arena()

    @classmethod
    def make_fully_connected(cls, state_dim: int, action_dim: int, layers: List[int],
                             activations: List[str], num_atoms: Optional[int] = None,
                             use_batch_norm: bool = False):
        """dueling_q_network.py:48-90"""
        assert len(layers) > 0, "Must have at least one layer"
        if use_batch_norm:
            raise NotImplementedError("dueling head with batch norm is out of scope")
        state_embedding_dim = layers[-1]
        assert state_embedding_dim % 2 == 0, "The last size must be divisible by 2"
        shared_network = FullyConnectedDQN(state_dim, state_embedding_dim, sizes=layers[:-1],
                                           activations=activations[:-1], normalized_output=True)
        advantage_network = FullyConnectedDQN(state_embedding_dim, action_dim,
                                              sizes=[state_embedding_dim // 2],
                                              activations=activations[-1:], num_atoms=num_atoms)
        value_network = FullyConnectedDQN(state_embedding_dim, 1,
                                          sizes=[state_embedding_dim // 2],
                                          activations=activations[-1:], num_atoms=num_atoms)
        return cls(shared_network=shared_network, advantage_network=advantage_network,
                   value_network=value_network)

    # ---- arena plumbing ------------------------------------------------------
    def _linears(self):
        s = [seq[0] for seq in self.shared_network.fc.dnn]
        a = [seq[0] for seq in self.advantage_network.fc.dnn]
        v = [seq[0] for seq in self.value_network.fc.dnn]
        return s, a, v

    def _build_arena(self, device=None):
        s, a, v = self._linears()
        sfc = self.shared_network.fc
        ar = DuelingArena(sfc.layers, [_lib.ACT[x] for x in sfc.activations],
                          _lib.ACT[self.advantage_network.fc.activations[0]], self.action_dim,
                          self.num_atoms or 1)
        dev = device if device is not None else s[0].weight.device
        flat = torch.zeros(ar.n, dtype=torch.float32, device=dev)
        E, H, A, N = ar.E, ar.H, ar.A * ar.N, ar.N
        Ls = len(s)
        views = []
        for l, lin in enumerate(s):
            views.append((lin, ar.weight_view(flat, l), ar.bias_view(flat, l)))
        wst = flat[ar.w_off[Ls]: ar.w_off[Ls] + 2 * H * E].view(2 * H, E)
        bst = flat[ar.b_off[Ls]: ar.b_off[Ls] + 2 * H]
        views.append((a[0], wst[:H], bst[:H]))
        views.append((v[0], wst[H:], bst[H:]))
        views.append((a[1], flat[ar.o_wa: ar.o_wa + A * H].view(A, H), flat[ar.o_ba: ar.o_ba + A]))
        views.append((v[1], flat[ar.o_wv: ar.o_wv + N * H].view(N, H), flat[ar.o_bv: ar.o_bv + N]))
        for lin, w, b in views:
            w.copy_(lin.weight.data.to(dev, torch.float32))
            b.copy_(lin.bias.data.to(dev, torch.float32))
            lin.weight.data = w
            lin.bias.data = b
            lin.weight._rb200_arena = ar
            lin.bias._rb200_arena = ar
        ar.flat = flat
        self._arena = ar
        if flat.is_cuda:
            ar.refresh()

    @property
    def arena(self) -> DuelingArena:
        return self._arena

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)  # moves the parameters (sub-networks re-flatten themselves)
        self._build_arena()          # ... and gather them into the dueling arena again
        return self

    def __deepcopy__(self, memo):
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k == "_arena":
                continue
            new.__dict__[k] = copy.deepcopy(v, memo)
        new._build_arena()
        return new

    # ---- forward ---------------------------------------------------------------
    def input_prototype(self):
        return self.shared_network.input_prototype()

    def _head_desc(self, value: bool) -> _lib.MlpT:
        """Descriptor of one head ([E -> H -> A or 1]) over the TRUE parameters in the arena."""
        ar = self._arena
        Ls = len(self.shared_network.fc.dnn)
        d = _lib.MlpT()
        d.n_layers = 2
        d.dims[0], d.dims[1], d.dims[2] = ar.E, ar.H, (ar.N if value else ar.A * ar.N)
        d.act[0], d.act[1] = ar.acts[Ls], _lib.ACT["linear"]
        d.w_off[0] = ar.w_off[Ls] + (ar.H * ar.E if value else 0)
        d.b_off[0] = ar.b_off[Ls] + (ar.H if value else 0)
        d.w_off[1] = ar.o_wv if value else ar.o_wa
        d.b_off[1] = ar.o_bv if value else ar.o_ba
        d.params = ar.flat.data_ptr()
        d.n_params = ar.n
        return d

    def _run(self, desc, x, out_dim):
        out = torch.empty(x.shape[0], out_dim, dtype=torch.float32, device=x.device)
        run_mlp(desc, x, out)
        return out

    def _get_values(self, state: rlt.FeatureData):
        """(value, raw_advantage, advantage, q_value) evaluated head by head on the true
        parameters (dueling_q_network.py:92-103); inspection path, three launches."""
        x = state.float_features
        require_cuda(x, "DuelingQNetwork._get_values")
        x = x.contiguous().float()
        ar = self._arena
        shared = self._run(ar.desc(len(self.shared_network.fc.dnn)), x, ar.E)
        value = self._run(self._head_desc(True), shared, ar.N)
        raw_advantage = self._run(self._head_desc(False), shared, ar.A * ar.N)
        if self.num_atoms is not None:  # (B, 1, N) and (B, A, N): fully_connected_network.py:215-217
            value = value.view(-1, 1, ar.N)
            raw_advantage = raw_advantage.view(-1, ar.A, ar.N)
        reduce_over = tuple(range(1, raw_advantage.dim()))
        advantage = raw_advantage - raw_advantage.mean(dim=reduce_over, keepdim=True)
        return value, raw_advantage, advantage, value + advantage

    def forward(self, state: rlt.FeatureData,
                possible_actions_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        x = state.float_features
        require_cuda(x, "DuelingQNetwork.forward")
        x = x.contiguous().float()
        ar = self._arena
        ar.refresh()
        R = ar.A * ar.N
        out = torch.empty(x.shape[0], R, dtype=torch.float32, device=x.device)
        if R > 256:  # wide head (atoms): fused trunk + 2-D tiled head, as FullyConnectedDQN does
            h = torch.empty(x.shape[0], ar.dims[-2], dtype=torch.float32, device=x.device)
            ar.forward_wide(x, out, h)
        else:
            ar.forward(x, out)
        if self.num_atoms is not None:
            out = out.view(-1, ar.A, ar.N)
        if possible_actions_mask is not None:
            # subtract a huge value from impossible actions (dueling_q_network.py:119-124)
            out = out + (1 - possible_actions_mask.float()) * INVALID_ACTION_CONSTANT
        return out
