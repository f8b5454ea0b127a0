"""Optimizer config surface of the reference (reagent/optimizer/union.py:52-64,
optimizer.py:47-85, uninferrable_optimizers.py:23-33, 70-78): `Optimizer__Union.default()` is
Adam; `make_optimizer_scheduler(params)` returns {"optimizer": ...}.  Adam and AdamW have a
fused sm_90a kernel (SURVEY.md 8a O2); other members of the reference's union raise."""
from dataclasses import dataclass, field
from typing import List, Tuple

from .fused_adam import FusedAdam, FusedAdamW


@dataclass(frozen=True)
class Adam:
    lr: float = 0.001
    betas: Tuple[float, float] = (0.9, 0.999)
    eps: float = 1e-08
    weight_decay: float = 0
    amsgrad: bool = False
    lr_schedulers: List = field(default_factory=list)

    def make_optimizer_scheduler(self, params):
        assert len(self.lr_schedulers) == 0, "lr schedulers are out of scope of the fused path"
        opt = FusedAdam(params, lr=self.lr, betas=tuple(self.betas), eps=self.eps,
                        weight_decay=self.weight_decay, amsgrad=self.amsgrad)
        return {"optimizer": opt}


@dataclass(frozen=True)
class AdamW:
    lr: float = 0.001
    betas: Tuple[float, float] = (0.9, 0.999)
    eps: float = 1e-08
    weight_decay: float = 0.01
    amsgrad: bool = False
    lr_schedulers: List = field(default_factory=list)

    def make_optimizer_scheduler(self, params):
        assert len(self.lr_schedulers) == 0, "lr schedulers are out of scope of the fused path"
        opt = FusedAdamW(params, lr=self.lr, betas=tuple(self.betas), eps=self.eps,
                         weight_decay=self.weight_decay, amsgrad=self.amsgrad)
        return {"optimizer": opt}


classes = {"Adam": Adam, "AdamW": AdamW}


class Optimizer__Union:
    def __init__(self, **kwargs):
        if len(kwargs) != 1:
            raise ValueError("Optimizer__Union takes exactly one member, e.g. Adam=...")
        (name, value), = kwargs.items()
        if name not in classes:
            raise NotImplementedError(
                f"optimizer {name!r} has no fused sm_90a kernel; supported: {sorted(classes)}")
        if isinstance(value, dict):
            value = classes[name](**value)
        self.selected_field = name
        self.value = value

    @classmethod
    def default(cls, **kwargs):
        return cls(Adam=Adam()) if kwargs == {} else cls(Adam=Adam(**kwargs))

    def make_optimizer_scheduler(self, params):
        return self.value.make_optimizer_scheduler(params)
