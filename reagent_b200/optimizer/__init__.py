from .fused_adam import FusedAdam, FusedAdamW  # noqa: F401
from .soft_update import SoftUpdate  # noqa: F401
from .union import Adam, AdamW, Optimizer__Union  # noqa: F401

__all__ = ["Optimizer__Union", "SoftUpdate", "FusedAdam", "FusedAdamW", "Adam", "AdamW"]
