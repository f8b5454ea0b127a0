"""FullyConnectedNetwork / FloatFeatureFullyConnected with the same constructor arguments,
sub-module names, initialisation and forward semantics as the reference
(reagent/models/fully_connected_network.py:21-23, :67-217), restricted to the in-scope
layer set (Linear + activation; BN / LN / dropout / residual raise NotImplementedError).
forward() is ONE fused CUDA launch over row tiles (rb200_mlp_forward)."""
import copy
import math
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.init as init

from .. import _lib
from ..core import types as rlt
from .arena import ParamArena, flatten_linears
from .base import ModelBase, require_cuda

ACTIVATION_MAP = {
    "tanh": nn.Tanh,
    "relu": nn.ReLU,
    "leaky_relu": nn.LeakyReLU,
    "linear": nn.Identity,
    "sigmoid": nn.Sigmoid,
    "softplus": nn.Softplus,
}


def gaussian_fill_w_gain(tensor, gain, dim_in, min_std=0.0) -> None:
    """Gaussian initialization with gain (fully_connected_network.py:21-23)."""
    init.normal_(tensor, mean=0, std=max(gain * math.sqrt(1 / dim_in), min_std))


class FullyConnectedNetwork(ModelBase):
    def __init__(
        self,
        layers,
        activations,
        *,
        use_batch_norm: bool = False,
        min_std: float = 0.0,
        dropout_ratio: float = 0.0,
        use_layer_norm: bool = False,
        normalize_output: bool = False,
        orthogonal_init: bool = False,
        use_skip_connections: bool = False,
    ) -> None:
        super().__init__()
        if use_batch_norm or use_layer_norm or dropout_ratio > 0.0 or use_skip_connections:
            raise NotImplementedError(
                "reagent_b200 covers the Linear+activation layer set of the hot path; "
                "batch/layer norm, dropout and skip connections are out of scope (SURVEY.md M1)")
        self.input_dim = layers[0]
        assert len(layers) == len(activations) + 1, (
            f"Invalid number of layers {len(layers)} and activations {len(activations)}. "
            "Number of layers needs to be 1 + number of activations")
        modules: List[nn.Module] = []
        for (in_dim, out_dim), activation in zip(zip(layers, layers[1:]), activations):
            if activation not in _lib.ACT:
                raise NotImplementedError(f"activation {activation!r} has no CUDA kernel")
            linear = nn.Linear(in_dim, out_dim)
            try:
                gain = torch.nn.init.calculate_gain(activation)
            except ValueError:
                gain = 1.0
            if orthogonal_init:
                nn.init.orthogonal_(linear.weight.data, gain=gain)
            else:
                gaussian_fill_w_gain(linear.weight, gain=gain, dim_in=in_dim, min_std=min_std)
            init.constant_(linear.bias, 0)
            modules.append(nn.Sequential(linear, ACTIVATION_MAP[activation]()))
        self.dnn = nn.Sequential(*modules)
        self.layers = list(layers)
        self.activations = list(activations)
        self._arena = ParamArena(self.layers, [_lib.ACT[a] for a in self.activations])
        flatten_linears(self._linears(), self._arena)

    # ---- arena plumbing ----------------------------------------------------
    def _linears(self):
        return [seq[0] for seq in self.dnn]

    @property
    def arena(self) -> ParamArena:
        return self._arena

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        # parameters were moved one by one: gather them into a fresh flat buffer again
        flatten_linears(self._linears(), self._arena)
        return self

    def __deepcopy__(self, memo):
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k == "_arena":
                continue
            new.__dict__[k] = copy.deepcopy(v, memo)
        new._arena = ParamArena(self.layers, [_lib.ACT[a] for a in self.activations])
        flatten_linears(new._linears(), new._arena)
        return new

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)  # copies in place -> views stay valid
        return out

    # ---- forward -------------------------------------------------------------
    def input_prototype(self):
        return torch.randn(1, self.input_dim)

    def forward_cat(self, x0: torch.Tensor, x1: Optional[torch.Tensor] = None) -> torch.Tensor:
        """out = MLP(cat(x0, x1)) as one fused launch."""
        require_cuda(x0, type(self).__name__ + ".forward")
        x0 = x0.contiguous().float()
        if x1 is not None:
            x1 = x1.contiguous().float()
        B = x0.shape[0]
        out = torch.empty(B, self.layers[-1], dtype=torch.float32, device=x0.device)
        if self.layers[-1] <= 1024:
            self._arena.forward(x0, out, x1=x1)
            return out
        # wide head (e.g. QR-DQN's A*N outputs): trunk as one fused launch, head 2-D tiled
        h = x0 if x1 is None else torch.cat((x0, x1), dim=1)
        trunk = (torch.empty(B, self.layers[-2], dtype=torch.float32, device=x0.device)
                 if len(self.layers) > 2 else None)
        self._arena.forward_wide(h, out, trunk)
        return out

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        return self.forward_cat(input)


class FloatFeatureFullyConnected(ModelBase):
    """fully_connected_network.py:166-217"""

    def __init__(
        self,
        state_dim,
        output_dim,
        sizes,
        activations,
        *,
        output_activation: str = "linear",
        num_atoms: Optional[int] = None,
        use_batch_norm: bool = False,
        dropout_ratio: float = 0.0,
        normalized_output: bool = False,
        use_layer_norm: bool = False,
    ):
        super().__init__()
        assert state_dim > 0, "state_dim must be > 0, got {}".format(state_dim)
        assert output_dim > 0, "output_dim must be > 0, got {}".format(output_dim)
        self.state_dim = state_dim
        self.output_dim = output_dim
        assert len(sizes) == len(activations), (
            "The numbers of sizes and activations must match; got {} vs {}".format(
                len(sizes), len(activations)))
        self.num_atoms = num_atoms
        self.fc = FullyConnectedNetwork(
            [state_dim] + list(sizes) + [output_dim * (num_atoms or 1)],
            list(activations) + [output_activation],
            use_batch_norm=use_batch_norm,
            dropout_ratio=dropout_ratio,
            normalize_output=normalized_output,
            use_layer_norm=use_layer_norm,
        )

    @property
    def arena(self):
        return self.fc.arena

    def input_prototype(self):
        return rlt.FeatureData(self.fc.input_prototype())

    def forward(self, state: rlt.FeatureData) -> torch.Tensor:
        float_features = state.float_features
        x = self.fc(float_features)
        if self.num_atoms is not None:
            x = x.view(float_features.shape[0], self.action_dim, self.num_atoms)
        return x
