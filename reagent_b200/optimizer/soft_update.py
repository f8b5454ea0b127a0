"""SoftUpdate pseudo-optimizer: target = tau*source + (1-tau)*target
(reagent/optimizer/soft_update.py:9-71), one CUDA launch per (target, source) network."""
import torch

from .. import _lib
from ..models.arena import arena_of


class SoftUpdate(torch.optim.Optimizer):
    def __init__(self, target_params, source_params, tau: float = 0.1) -> None:
        target_params = list(target_params)
        source_params = list(source_params)
        if len(target_params) != len(source_params):
            raise ValueError("target and source must have the same number of parameters")
        for t_param, s_param in zip(target_params, source_params):
            if t_param.shape != s_param.shape:
                raise ValueError("The shape of target parameter doesn't match that of the source")
        params = target_params + source_params
        defaults = dict(tau=tau, lr=1.0)
        super().__init__(params, defaults)
        for group in self.param_groups:
            tau = group["tau"]
            if tau > 1.0 or tau < 0.0:
                raise ValueError(f"tau should be in [0.0, 1.0]; got {tau}")
        # group the parameter pairs by network arena (in order of first appearance)
        self._pairs = []
        seen = {}
        for t, s in zip(target_params, source_params):
            ta, sa = arena_of([t]), arena_of([s])
            key = (id(ta), id(sa))
            if key not in seen:
                seen[key] = True
                self._pairs.append((ta, sa))

    @classmethod
    def make_optimizer_scheduler(cls, target_params, source_params, tau):
        su = cls(target_params, source_params, tau)
        return {"optimizer": su}

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for ta, sa in self._pairs:
            if ta is not sa:  # aliased target: soft_update.py:64-67
                self.update(ta, sa)
        return loss

    def update(self, ta, sa):
        """target arena `ta` <- tau * source arena `sa` + (1 - tau) * `ta`."""
        tau = self.param_groups[0]["tau"]
        _lib.check(
            _lib.lib().rb200_soft_update(ta.flat.data_ptr(), sa.flat.data_ptr(), ta.n,
                                         float(tau), float(1.0 - tau), _lib.cur_stream()),
            "rb200_soft_update")
        ta.data_epoch = getattr(ta, "data_epoch", 0) + 1

    def zero_grad(self, set_to_none: bool = True):
        pass
