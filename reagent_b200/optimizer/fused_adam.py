"""Adam and AdamW over a flat parameter arena, one fused CUDA launch per step (K3).

Numerics follow torch.optim.Adam's single-tensor path, which is what the reference gets
from `Optimizer__Union.default()` -> `torch.optim.Adam(lr=1e-3, betas=(0.9, 0.999),
eps=1e-8, weight_decay=0, amsgrad=False)` (reagent/optimizer/optimizer.py:64-85,
reagent/optimizer/uninferrable_optimizers.py:23-33).  Gradients are NOT read from
`p.grad`: the trainer's fused backward leaves split-K partials in `arena.gpart`, which the
kernel sums in a fixed order (deterministic) before the update.

FusedAdamW is the counterpart of torch.optim.AdamW (decoupled weight decay, optional AMSGrad),
which the reference's CartPole QR-DQN / C51 configurations select with
`AdamW: {lr: 0.001, amsgrad: true}` (reagent/optimizer/uninferrable_optimizers.py:70-78).
"""
from typing import Optional

import torch

from .. import _lib
from ..models.arena import ParamArena, ScalarArena, arena_of


_TORCH_FLAGS = dict(amsgrad=False, maximize=False, foreach=None, capturable=False,
                    differentiable=False, fused=None, decoupled_weight_decay=False)
# group flags of torch.optim.Adam that change the update rule; FusedAdam has none of them
# (FusedAdamW has decoupled_weight_decay and amsgrad)
_UNSUPPORTED_FLAGS = ("amsgrad", "maximize", "decoupled_weight_decay")


class FusedAdam(torch.optim.Optimizer):
    _decoupled = False  # AdamW's decoupled weight decay (FusedAdamW)

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                 amsgrad=False, maximize=False, **unused):
        if amsgrad:
            raise NotImplementedError("FusedAdam has no amsgrad (reference default is False); "
                                      "FusedAdamW has")
        self._setup(params, lr, betas, eps, weight_decay, amsgrad, maximize)

    def _setup(self, params, lr, betas, eps, weight_decay, amsgrad, maximize):
        if maximize:
            raise NotImplementedError("maximize has no fused kernel (reference default is False)")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        params = list(params)
        # torch.optim.Adam's (AdamW's) group keys, with the values this kernel implements, so
        # that checkpoints move between the two optimizers in either direction
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                        **dict(_TORCH_FLAGS, amsgrad=bool(amsgrad),
                               decoupled_weight_decay=self._decoupled))
        super().__init__(params, defaults)
        if len(self.param_groups) != 1:
            raise NotImplementedError(f"{type(self).__name__} takes one parameter group (one network)")
        self.amsgrad = bool(amsgrad)
        ps = self.param_groups[0]["params"]
        if len(ps) == 1 and getattr(ps[0], "_rb200_arena", None) is None:
            ScalarArena(ps[0])  # stand-alone parameter such as SAC's log_alpha
        self.arena: ParamArena = arena_of(ps)
        self._flat_id = None
        self._alloc_state()

    # ------------------------------------------------------------------
    def _alloc_state(self):
        flat = self.arena.flat
        self._flat_id = flat.data_ptr()
        dev = flat.device
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        # AMSGrad's running maximum of exp_avg_sq, with the arena's layout
        self.max_exp_avg_sq = torch.zeros_like(flat) if self.amsgrad else None
        self.step_t = torch.zeros(1, dtype=torch.int64, device=dev)
        self._counter = torch.zeros(1, dtype=torch.int32, device=dev)

    def _ensure_state(self):
        flat = self.arena.flat
        if flat.data_ptr() != self._flat_id:
            # the model was moved (e.g. .cuda()) after the optimizer was built: follow it
            old = (self.exp_avg, self.exp_avg_sq, self.step_t, self.max_exp_avg_sq)
            self._alloc_state()
            self.exp_avg.copy_(old[0].to(flat.device))
            self.exp_avg_sq.copy_(old[1].to(flat.device))
            self.step_t.copy_(old[2].to(flat.device))
            if self.amsgrad:
                self.max_exp_avg_sq.copy_(old[3].to(flat.device))

    @property
    def num_steps(self) -> int:
        return int(self.step_t.item())

    # ------------------------------------------------------------------
    @torch.no_grad()
    def fused_step(self, target: Optional[ParamArena] = None, tau: float = 0.0,
                   grad: Optional[torch.Tensor] = None, grad_scale: float = 1.0,
                   exp_out: Optional[torch.Tensor] = None, tc_pack=None, dp=None):
        """Adam step (+ Polyak update of `target` with the NEW parameters when given).
        `tc_pack = (pack_tensor, do_backward)`: also write the tensor-core weight images of the
        updated network and target for the next rb200_dqn_td_step_tc (needs `target`).
        `dp`: a training.data_parallel.P2PExchange -- the gradient exchange between the ranks is
        fused into this launch (peer-to-peer stores over NVLink, summed in rank order, scaled
        by 1/world); `grad` must then be this rank's own split-K partials (the default)."""
        self._ensure_state()
        a = self.arena
        if grad is None:
            if a.gpart is None or not a.grad_ready:
                raise _lib.Rb200Error(
                    f"{type(self).__name__}.step(): no gradient partials for this network -- run the "
                    "trainer's train_step_gen/next() (fused backward) first")
            grad = a.gpart
        splits = grad.shape[0] if grad.dim() == 2 else 1
        g = self.param_groups[0]
        args = _lib.AdamArgsT()
        args.params = a.flat.data_ptr()
        args.grad = grad.data_ptr()
        args.splits = splits
        args.n = a.n
        args.exp_avg = self.exp_avg.data_ptr()
        args.exp_avg_sq = self.exp_avg_sq.data_ptr()
        args.step = self.step_t.data_ptr()
        args.block_counter = self._counter.data_ptr()
        args.lr = float(g["lr"])
        args.beta1, args.beta2 = float(g["betas"][0]), float(g["betas"][1])
        args.eps = float(g["eps"])
        args.weight_decay = float(g["weight_decay"])
        args.grad_scale = float(grad_scale)
        args.decoupled_weight_decay = int(self._decoupled)
        args.amsgrad = int(self.amsgrad)
        args.max_exp_avg_sq = self.max_exp_avg_sq.data_ptr() if self.amsgrad else None
        if target is not None:
            if target.n != a.n:
                raise ValueError("target / source arenas differ in size")
            args.target = target.flat.data_ptr()
            args.tau = float(tau)
            args.one_minus_tau = float(1.0 - tau)
        else:
            args.target = None
            args.tau = 0.0
            args.one_minus_tau = 1.0
        args.exp_out = None if exp_out is None else exp_out.data_ptr()
        args.dp_world = 1
        if dp is not None and dp.world > 1:
            recv, flags, stride, maxb = dp.slice_for(id(self), a.n)
            args.dp_world, args.dp_rank = dp.world, dp.rank
            args.dp_recv, args.dp_flags = recv.data_ptr(), flags.data_ptr()
            args.dp_stride, args.dp_max_blocks = stride, maxb
            args.grad_scale = float(grad_scale) / dp.world
        desc = None
        if tc_pack is not None and target is not None:
            import ctypes as C

            desc = a.desc()  # kept alive until the launch returns
            args.tc_net = C.pointer(desc)
            args.tc_pack_ws = tc_pack[0].data_ptr()
            args.tc_pack_ws_bytes = tc_pack[0].numel()
            args.tc_do_backward = int(tc_pack[1])
        _lib.check(_lib.lib().rb200_adam_soft_update(args, _lib.cur_stream()),
                   "rb200_adam_soft_update")
        a.grad_ready = False
        # every library write to an arena bumps its epoch (caches keyed on parameter contents)
        a.data_epoch = getattr(a, "data_epoch", 0) + 1
        if target is not None:
            target.data_epoch = getattr(target, "data_epoch", 0) + 1
        return desc is not None

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.fused_step()
        return loss

    def zero_grad(self, set_to_none: bool = True):
        # gradients live in arena.gpart and are overwritten by every fused backward
        for p in self.param_groups[0]["params"]:
            p.grad = None

    # state_dict in torch.optim.Adam's (AdamW's) shape: per-parameter views of the flat moments
    def state_dict(self):
        self._ensure_state()
        sd = super().state_dict()
        a = self.arena
        state = {}
        ps = self.param_groups[0]["params"]
        flat = a.flat
        base = flat.data_ptr()
        for i, p in enumerate(ps):
            off = (p.data_ptr() - base) // 4
            n = p.numel()
            state[i] = {
                "step": self.step_t.detach().clone().float().reshape(()),
                "exp_avg": self.exp_avg[off:off + n].view_as(p).clone(),
                "exp_avg_sq": self.exp_avg_sq[off:off + n].view_as(p).clone(),
            }
            if self.amsgrad:
                state[i]["max_exp_avg_sq"] = self.max_exp_avg_sq[off:off + n].view_as(p).clone()
        sd["state"] = state
        return sd

    def _check_group_flags(self, group):
        for k in _UNSUPPORTED_FLAGS:
            if group.get(k, False):
                raise NotImplementedError(
                    f"state dict has {k}=True, which has no fused kernel (reference default "
                    "is False)")

    def load_state_dict(self, state_dict):
        for group in state_dict.get("param_groups", []):
            self._check_group_flags(group)
        self._ensure_state()
        ps = self.param_groups[0]["params"]
        base = self.arena.flat.data_ptr()
        st = state_dict.get("state", {})
        for i, p in enumerate(ps):
            if i not in st:
                continue
            off = (p.data_ptr() - base) // 4
            n = p.numel()
            self.exp_avg[off:off + n].copy_(st[i]["exp_avg"].reshape(-1))
            self.exp_avg_sq[off:off + n].copy_(st[i]["exp_avg_sq"].reshape(-1))
            if self.amsgrad:
                self.max_exp_avg_sq[off:off + n].copy_(st[i]["max_exp_avg_sq"].reshape(-1))
            self.step_t.fill_(int(st[i]["step"]))
        for k in ("lr", "betas", "eps", "weight_decay"):
            if state_dict.get("param_groups"):
                self.param_groups[0][k] = state_dict["param_groups"][0].get(k, self.param_groups[0][k])


class FusedAdamW(FusedAdam):
    """torch.optim.AdamW (decoupled weight decay, weight_decay=0.01 by default, optional
    AMSGrad) on the fused K3 kernel.  `maximize` has no kernel and raises."""
    _decoupled = True

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                 amsgrad=False, maximize=False, **unused):
        self._setup(params, lr, betas, eps, weight_decay, amsgrad, maximize)

    def _check_group_flags(self, group):
        if group.get("maximize", False):
            raise NotImplementedError("state dict has maximize=True, which has no fused kernel")
        if not group.get("decoupled_weight_decay", False):
            raise ValueError("state dict has decoupled_weight_decay=False (torch.optim.Adam's); "
                             "load it into FusedAdam")
        if bool(group.get("amsgrad", False)) != self.amsgrad:
            raise ValueError(f"state dict has amsgrad={group.get('amsgrad')}, this optimizer "
                             f"was built with amsgrad={self.amsgrad}")
