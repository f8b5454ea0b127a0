"""Flat parameter arena shared by every model in this package.

Each network keeps ordinary `nn.Linear` sub-modules (so `state_dict()` keys and shapes are
the reference's: `fc.dnn.{i}.0.weight`, reagent/models/fully_connected_network.py:101-153)
but their `.data` are views into ONE contiguous fp32 buffer laid out
[W0, b0, W1, b1, ...] with every tensor starting on a 16-byte boundary.  The CUDA kernels
see the arena (base pointer + offsets, `rb200_mlp_t`); Adam, the Polyak update and the
gradient all-reduce are single launches over it.
"""
import ctypes as C
from typing import List, Optional

import torch
import torch.nn as nn

from .. import _lib


def _align4(n: int) -> int:
    return (n + 3) & ~3


class ParamArena:
    """The flat buffer + layout of one network (or of one stand-alone parameter)."""

    def __init__(self, dims: List[int], acts: List[int]):
        assert len(dims) == len(acts) + 1
        assert 1 <= len(acts) <= _lib.MAX_LAYERS, f"at most {_lib.MAX_LAYERS} layers are supported"
        self.dims = list(dims)
        self.acts = list(acts)
        self.w_off, self.b_off = [], []
        off = 0
        for i in range(len(acts)):
            self.w_off.append(off)
            off = _align4(off + dims[i] * dims[i + 1])
            self.b_off.append(off)
            off = _align4(off + dims[i + 1])
        self.n = off
        self.flat: Optional[torch.Tensor] = None
        # filled by the trainer that owns the update of this arena
        self.gpart: Optional[torch.Tensor] = None   # [splits, n] gradient partials
        self.grad_ready = False
        self._desc = None

    # -- hooks for arenas with derived regions (models/dueling_q_network.py) ------
    def refresh(self):
        """Bring derived parameters up to date before the kernels read the arena (no-op here)."""

    def finish_grads(self):
        """Map gradients of derived parameters back onto the true ones (no-op here)."""

    # -- views ---------------------------------------------------------------
    def weight_view(self, flat, l):
        o, i = self.dims[l + 1], self.dims[l]
        return flat[self.w_off[l]: self.w_off[l] + o * i].view(o, i)

    def bias_view(self, flat, l):
        o = self.dims[l + 1]
        return flat[self.b_off[l]: self.b_off[l] + o]

    def layer_ptrs(self, l):
        """Device pointers of layer l's weight and bias in the current flat buffer."""
        f = self.flat.data_ptr()
        return f + 4 * self.w_off[l], f + 4 * self.b_off[l]

    def desc(self, n_layers=None) -> _lib.MlpT:
        """ctypes descriptor for the current flat buffer (optionally only the first
        `n_layers` layers, e.g. the trunk below a wide head)."""
        assert self.flat is not None
        L = len(self.acts) if n_layers is None else n_layers
        d = _lib.MlpT()
        d.n_layers = L
        for i, v in enumerate(self.dims[: L + 1]):
            d.dims[i] = v
        for i, a in enumerate(self.acts[:L]):
            d.act[i] = a
            d.w_off[i] = self.w_off[i]
            d.b_off[i] = self.b_off[i]
        d.params = self.flat.data_ptr()
        d.n_params = self.n
        return d

    # -- launches (the library is looked up per call, so a wrapped entry point takes effect) --
    def forward(self, x, out, *, n_layers=None, x1=None, save=None):
        """out = MLP(cat(x, x1)) over the first `n_layers` layers as one fused launch; `save`
        (a NetWorkspace) keeps the activations the backward reads."""
        run_mlp(self.desc(n_layers), x, out, x1=x1, save=save)

    def forward_wide(self, x, out, trunk_out, save=None):
        """out = MLP(x) for a head too wide for the fused row tiles: the trunk (all layers but
        the last) as one fused launch into `trunk_out` [B, dims[-2]] (None for a one-layer
        network), then the last layer as a 2-D tiled linear."""
        L = len(self.acts)
        h = x
        if L > 1:
            self.forward(x, trunk_out, n_layers=L - 1, save=save)
            h = trunk_out
        W, b = self.layer_ptrs(L - 1)
        rc = _lib.lib().rb200_linear_forward(W, b, self.acts[L - 1], self.dims[L - 1], self.dims[L],
                                             h.data_ptr(), x.shape[0], out.data_ptr(),
                                             _lib.cur_stream())
        _lib.check(rc, "rb200_linear_forward(head)")

    def backward(self, ws, batch: int, n_layers=None):
        """dZ chain of the first `n_layers` layers from the dZ of the last of them (in `ws`)."""
        L = len(self.acts) if n_layers is None else n_layers
        rc = _lib.lib().rb200_mlp_backward(self.desc(n_layers), ws.dz[L - 1].data_ptr(), batch,
                                           ws.c, _lib.cur_stream())
        if rc == _lib.E_SMEM:
            # hidden layers too wide for the fused row tile (it keeps three of them in shared
            # memory; [1024, 1024] does not fit): the same chain one layer per launch.  Nothing
            # was launched by the refused call.
            cache = self.__dict__.setdefault("_dx_scratch", {})
            for l in range(L - 1, 0, -1):
                self.layer_backward_dx(l, ws, batch, cache)
            return
        _lib.check(rc, "rb200_mlp_backward")

    def layer_backward_dx(self, l: int, ws, batch: int, cache: dict):
        """dZ of layer l - 1 from the dZ of layer l: dz[l-1] = (dz[l] . W_l) * act'(h[l-1])
        (torch.nn.functional.linear's backward w.r.t. its input).  Wide layers take the wgmma
        split-K path, which needs a scratch buffer kept in `cache`."""
        lib, st = _lib.lib(), _lib.cur_stream()
        K, N = self.dims[l], self.dims[l + 1]
        W, _ = self.layer_ptrs(l)
        dz, h, out = ws.dz[l], ws.hidden[l - 1], ws.dz[l - 1]
        key = ("dx_scratch", K, N, batch)
        if key not in cache:
            nbytes = int(lib.rb200_linear_backward_dx_tc_scratch_bytes(K, N, batch))
            cache[key] = torch.empty(nbytes // 4, device=self.flat.device) if nbytes else None
        scratch = cache[key]
        if scratch is not None:
            rc = lib.rb200_linear_backward_dx_tc(W, K, N, dz.data_ptr(), h.data_ptr(),
                                                 self.acts[l - 1], batch, out.data_ptr(),
                                                 scratch.data_ptr(), scratch.numel() * 4, st)
            _lib.check(rc, "rb200_linear_backward_dx_tc")
        else:
            rc = lib.rb200_linear_backward_dx(W, K, N, dz.data_ptr(), h.data_ptr(),
                                              self.acts[l - 1], batch, out.data_ptr(), st)
            _lib.check(rc, "rb200_linear_backward_dx")


def run_mlp(desc: _lib.MlpT, x, out, x1=None, save=None):
    """One fused MLP forward over `desc`: out = MLP(cat(x, x1)) for the x.shape[0] rows of x."""
    rc = _lib.lib().rb200_mlp_forward(desc, x.data_ptr(), x.shape[1], _lib.ptr(x1),
                                      0 if x1 is None else x1.shape[1], x.shape[0], out.data_ptr(),
                                      None if save is None else save.c, _lib.cur_stream())
    _lib.check(rc, "rb200_mlp_forward")


def run_mlp_tiled(arenas, state, actions, num_tiled: int, outs):
    """outs[n][r] = arenas[n](cat(state[r // num_tiled], actions[r])) for one or two arenas of
    identical shape (online and target), as ONE launch over a shared input tile; bit-equal to
    run_mlp on the materialised cat(state.repeat_interleave(num_tiled), actions)."""
    assert len(arenas) == len(outs) in (1, 2)
    # the C ABI takes no row count for `actions` or the outputs: check every shape here
    B, M = state.shape[0], int(num_tiled)
    dev = state.device
    named = [("state", state), ("actions", actions)] + [(f"outs[{i}]", o) for i, o in enumerate(outs)]
    for name, t in named:
        assert t.dim() == 2 and t.dtype == torch.float32 and t.is_cuda and t.device == dev, (
            f"{name}: expected a 2-D float32 CUDA tensor on {dev}, "
            f"got {t.dtype} {tuple(t.shape)} on {t.device}")
        assert t.is_contiguous(), f"{name} must be contiguous"
    assert M >= 1 and actions.shape[0] == B * M, (
        f"actions has {actions.shape[0]} rows, expected batch {B} * num_tiled {M}")
    assert state.shape[1] + actions.shape[1] == arenas[0].dims[0], (
        f"state width {state.shape[1]} + action width {actions.shape[1]} != {arenas[0].dims[0]}")
    for i, (a, o) in enumerate(zip(arenas, outs)):
        assert tuple(o.shape) == (B * M, a.dims[-1]), f"outs[{i}] shape {tuple(o.shape)}"
    d1 = arenas[1].desc() if len(arenas) == 2 else None
    rc = _lib.lib().rb200_mlp_forward_tiled(
        arenas[0].desc(), d1, state.data_ptr(), state.shape[1], actions.data_ptr(),
        actions.shape[1], state.shape[0], num_tiled, outs[0].data_ptr(),
        None if d1 is None else outs[1].data_ptr(), _lib.cur_stream())
    _lib.check(rc, "rb200_mlp_forward_tiled")


def flatten_linears(linears: List[nn.Linear], arena: ParamArena, device=None) -> torch.Tensor:
    """Move the Linear parameters into one flat buffer (keeping their values) and re-point
    `.data` at views of it.  Returns the flat tensor."""
    dev = device if device is not None else linears[0].weight.device
    flat = torch.zeros(arena.n, dtype=torch.float32, device=dev)
    for l, lin in enumerate(linears):
        w = arena.weight_view(flat, l)
        b = arena.bias_view(flat, l)
        w.copy_(lin.weight.data.to(dev, torch.float32))
        b.copy_(lin.bias.data.to(dev, torch.float32))
        lin.weight.data = w
        lin.bias.data = b
        lin.weight._rb200_arena = arena
        lin.bias._rb200_arena = arena
    arena.flat = flat
    arena.gpart = None
    arena.grad_ready = False
    return flat


def arena_of(params) -> ParamArena:
    """The arena a list of parameters belongs to (all must share one)."""
    params = list(params)
    if not params:
        raise ValueError("empty parameter list")
    a = getattr(params[0], "_rb200_arena", None)
    if a is None:
        raise ValueError(
            "parameter does not belong to a reagent_b200 network (no flat arena); "
            "build the network with reagent_b200.models / net_builder")
    for p in params:
        if getattr(p, "_rb200_arena", None) is not a:
            raise ValueError("parameters of one optimizer must come from ONE reagent_b200 network")
    return a


class ScalarArena(ParamArena):
    """Arena wrapping one stand-alone contiguous parameter (e.g. SAC's log_alpha).  `flat`
    follows the parameter when the owning module is moved between devices."""

    def __init__(self, param: torch.nn.Parameter):
        self.dims, self.acts, self.w_off, self.b_off = [], [], [], []
        self.n = param.numel()
        self._param = param
        self.gpart = None
        self.grad_ready = False
        param._rb200_arena = self

    @property
    def flat(self):
        return self._param.data.view(-1)

    @flat.setter
    def flat(self, v):
        pass
