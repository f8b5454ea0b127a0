"""ModelBase (reagent/models/base.py:14-62): target-network copy + arena re-flattening
after device moves."""
import copy

import torch
import torch.nn as nn

from .. import _lib
from ..core import types as rlt


class ModelBase(nn.Module):
    def input_prototype(self):
        raise NotImplementedError

    def feature_config(self):
        return None

    def get_target_network(self):
        """deepcopy of the network (reagent/models/base.py:34-41)."""
        return copy.deepcopy(self)

    def get_distributed_data_parallel_model(self):
        raise NotImplementedError


def require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise _lib.Rb200Error(
            f"{what}: reagent_b200 runs on CUDA (sm_90a) only; got a {t.device} tensor. "
            "There is no CPU fallback -- move the model and batch to the GPU.")
