"""CEMPlannerNetwork (reagent/models/cem_planner.py): plans the next action by simulating
trajectories with an ensemble of world models (MemoryNetworks) and refining the plan with the
cross-entropy method.

Each CEM iteration is one launch of rb200_cem_rollout (csrc/rb200_cem.cu), which rolls every
trajectory of the population through the horizon, sampling from the world model as the
reference does, and reduces the iteration on the device: elites and the fp64 mean / var update
(continuous actions), or the first-action tally (discrete actions).  A plan therefore needs no
host synchronisation until its action is read.

The random numbers of a plan are drawn up front into one device buffer (CEMNoise) with torch's
CUDA generator, so a plan is reproducible under torch.manual_seed.  The reference's own streams
(numpy, `random`, torch's CPU generator, scipy) are not reproduced.
"""
import math
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from .. import _lib
from ..core import types as rlt
from ..core.parameters import CONTINUOUS_TRAINING_ACTION_RANGE
from .world_model import MemoryNetwork

# truncnorm(-2, 2) by inversion: ndtri(PHI_LO + u * PHI_WIDTH), u ~ U[0, 1)
PHI_LO = 0.5 * math.erfc(math.sqrt(2.0))  # Phi(-2)
PHI_WIDTH = math.erf(math.sqrt(2.0))      # Phi(2) - Phi(-2)


def _nbytes(shape, dtype):
    n = 1
    for s in shape:
        n *= s
    return -(-n * torch.empty((), dtype=dtype).element_size() // 8) * 8


class CEMNoise:
    """Every random number of one plan, as typed views of ONE device buffer:
      model_idx   int32 [iters, P]          world model of each trajectory
      action_idx  int32 [P, H]              discrete: the action of each step
      truncnorm   fp64  [iters, P, H * A]   continuous: truncnorm(-2, 2) draws of the solutions
      step        fp32  [iters, P, H, S+2]  per step: mixture uniform | S normals | Bernoulli
                                            uniform
    Discrete plans have one iteration and no truncnorm; continuous plans have no action_idx."""

    def __init__(self, iters, P, H, A, S, num_models, discrete, device):
        self.iters, self.P, self.H, self.A, self.S = iters, P, H, A, S
        self.num_models, self.discrete = num_models, discrete
        layout = [("truncnorm", (iters, P, H * A), torch.float64, not discrete),
                  ("step", (iters, P, H, S + 2), torch.float32, True),
                  ("model_idx", (iters, P), torch.int32, True),
                  ("action_idx", (P, H), torch.int32, discrete)]
        total = sum(_nbytes(s, t) for _, s, t, on in layout if on)
        self.buffer = torch.empty(max(total, 8), dtype=torch.uint8, device=device)
        off = 0
        for name, shape, dtype, on in layout:
            view = None
            if on:
                n = _nbytes(shape, dtype)
                view = self.buffer[off: off + n].view(dtype)[:math.prod(shape)].view(shape)
                off += n
            setattr(self, name, view)

    @property
    def device(self):
        return self.buffer.device

    def fill_(self) -> "CEMNoise":
        """Draw every number from torch's default generator of the buffer's device, in a fixed
        order: model indices, action indices, truncated normals, step uniforms and normals."""
        self.model_idx.random_(0, self.num_models)
        if self.discrete:
            self.action_idx.random_(0, self.A)
        else:
            u = self.truncnorm.uniform_()
            torch.special.ndtri(u.mul_(PHI_WIDTH).add_(PHI_LO), out=u)
        self.step[..., 0].uniform_()
        self.step[..., 1:self.S + 1].normal_()
        self.step[..., self.S + 1].uniform_()
        return self

    def copy_(self, model_idx, step, action_idx=None, truncnorm=None) -> "CEMNoise":
        """Take the numbers from arrays or tensors of the shapes above (tests, goldens)."""
        self.model_idx.copy_(torch.as_tensor(model_idx).to(torch.int32))
        self.step.copy_(torch.as_tensor(step).to(torch.float32))
        if self.discrete:
            self.action_idx.copy_(torch.as_tensor(action_idx).to(torch.int32))
        else:
            self.truncnorm.copy_(torch.as_tensor(truncnorm).to(torch.float64))
        return self


@dataclass
class CEMPlan:
    """What one plan leaves on the device (views of the planner's workspace, overwritten by the
    next plan).  `action`: discrete, the int64 index [1]; continuous, the float64 first action
    [A] rescaled to CONTINUOUS_TRAINING_ACTION_RANGE.  `values` [iters, P] fp64 solution values,
    `elites` [iters, num_elites], `mean` / `var` [iters, H * A] after each update and
    `n_iters` [1] (continuous); `one_hot` [A] float32 (discrete)."""
    action: torch.Tensor
    one_hot: Optional[torch.Tensor]
    values: torch.Tensor
    elites: Optional[torch.Tensor]
    mean: Optional[torch.Tensor]
    var: Optional[torch.Tensor]
    n_iters: torch.Tensor


class _Workspace:
    def __init__(self, planner: "CEMPlannerNetwork", device):
        p = planner
        P, H, A, S, it = p.cem_pop_size, p.plan_horizon_length, p.action_dim, p.state_dim, p.iters
        HA = H * A
        z = lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype, device=device)  # noqa: E731
        self.device = device
        self.state = z(S, dtype=torch.float32)
        self.discount = torch.tensor([p.gamma ** j for j in range(H)], dtype=torch.float32,
                                     device=device)
        self.values = z(max(it, 1), P)
        self.done = z(1, dtype=torch.int32)
        self.n_iters = z(1, dtype=torch.int32)
        self.counter = z(1, dtype=torch.int32)
        self.noise = CEMNoise(it, P, H, A, S, len(p.mem_net_list), p.discrete_action, device)
        if p.discrete_action:
            self.action_out = z(1, dtype=torch.int64)
            self.one_hot = z(A, dtype=torch.float32)
        else:
            self.lower = torch.from_numpy(p.action_lower_bounds.astype(np.float64)).to(device)
            self.upper = torch.from_numpy(p.action_upper_bounds.astype(np.float64)).to(device)
            self.mean0 = (self.upper + self.lower) / 2
            self.var0 = (self.upper - self.lower) ** 2 / 16
            self.mean, self.var = z(HA), z(HA)
            self.mean_hist, self.var_hist = z(max(it, 1), HA), z(max(it, 1), HA)
            self.elites = z(max(it, 1), p.num_elites, dtype=torch.int32)
            self.orig_lower = p.orig_action_lower.to(device, torch.float64)
            self.orig_upper = p.orig_action_upper.to(device, torch.float64)


class CEMPlannerNetwork(nn.Module):
    def __init__(self, mem_net_list: List[MemoryNetwork], cem_num_iterations: int,
                 cem_population_size: int, ensemble_population_size: int, num_elites: int,
                 plan_horizon_length: int, state_dim: int, action_dim: int,
                 discrete_action: bool, terminal_effective: bool, gamma: float,
                 alpha: float = 0.25, epsilon: float = 0.001,
                 action_upper_bounds: Optional[np.ndarray] = None,
                 action_lower_bounds: Optional[np.ndarray] = None):
        super().__init__()
        if ensemble_population_size != 1:
            # the reference stores an array of ensemble_population_size sums into one float slot
            # of acc_rewards_of_all_solutions, which numpy refuses for any other value
            raise ValueError(f"CEMPlannerNetwork: ensemble_population_size must be 1 (got "
                             f"{ensemble_population_size}); the reference fails on any other "
                             "value")
        mem_net_list = list(mem_net_list)
        for net in mem_net_list:
            if not isinstance(net, MemoryNetwork):
                raise NotImplementedError("CEMPlannerNetwork plans with "
                                          "reagent_b200.models.MemoryNetwork world models; got "
                                          + type(net).__name__)
        shapes = {(n.state_dim, n.action_dim, n.num_hiddens, n.num_hidden_layers,
                   n.num_gaussians) for n in mem_net_list}
        if len(shapes) != 1:
            raise ValueError(f"CEMPlannerNetwork: the world models must share one shape, got "
                             f"{sorted(shapes)}")
        shape = shapes.pop()
        if shape[:2] != (state_dim, action_dim):
            raise ValueError(f"CEMPlannerNetwork: world models take state_dim, action_dim = "
                             f"{shape[:2]}, the planner {state_dim, action_dim}")
        _lib.check(_lib.lib().rb200_cem_check_shape(*shape, cem_population_size,
                                                    len(mem_net_list), plan_horizon_length,
                                                    num_elites), "CEMPlannerNetwork")
        self.mem_net_list = nn.ModuleList(mem_net_list)
        self.cem_num_iterations = cem_num_iterations
        self.cem_pop_size = cem_population_size
        self.ensemble_pop_size = ensemble_population_size
        self.num_elites = num_elites
        self.plan_horizon_length = plan_horizon_length
        self.state_dim = state_dim
        self.action_dim = action_dim
        self.terminal_effective = terminal_effective
        self.gamma = gamma
        self.alpha = alpha
        self.epsilon = epsilon
        self.discrete_action = discrete_action
        # the discrete planner is one pass of random shooting
        self.iters = 1 if discrete_action else cem_num_iterations
        if not discrete_action:
            assert ((action_upper_bounds is not None) and (action_lower_bounds is not None)
                    and (action_upper_bounds.shape == action_lower_bounds.shape == (action_dim,)))
            assert np.all(action_upper_bounds >= action_lower_bounds)
            self.action_upper_bounds = np.tile(action_upper_bounds, self.plan_horizon_length)
            self.action_lower_bounds = np.tile(action_lower_bounds, self.plan_horizon_length)
            self.orig_action_upper = torch.tensor(action_upper_bounds)
            self.orig_action_lower = torch.tensor(action_lower_bounds)
        self._ws: Optional[_Workspace] = None

    def new_noise(self, device) -> CEMNoise:
        """An unfilled noise buffer of this planner's shape."""
        return CEMNoise(self.iters, self.cem_pop_size, self.plan_horizon_length, self.action_dim,
                        self.state_dim, len(self.mem_net_list), self.discrete_action, device)

    def _workspace(self, device) -> _Workspace:
        if self._ws is None or self._ws.device != device:
            self._ws = _Workspace(self, device)
        return self._ws

    def _args(self, ws: _Workspace, noise: CEMNoise, dump) -> "_lib.CemArgsT":
        a = _lib.CemArgsT()
        a.net = self.mem_net_list[0].mdnrnn.args(1, 1)
        a.num_models = len(self.mem_net_list)
        for m, net in enumerate(self.mem_net_list):
            a.params[m] = _lib.ptr(net.arena.flat, ws.device)
        a.population, a.horizon, a.iters = self.cem_pop_size, self.plan_horizon_length, self.iters
        a.num_elites, a.discrete = self.num_elites, int(self.discrete_action)
        a.terminal_effective = int(self.terminal_effective)
        a.alpha, a.epsilon = self.alpha, self.epsilon
        a.state, a.discount = ws.state.data_ptr(), ws.discount.data_ptr()
        a.model_idx, a.step_noise = noise.model_idx.data_ptr(), noise.step.data_ptr()
        a.values, a.done, a.n_iters = ws.values.data_ptr(), ws.done.data_ptr(), ws.n_iters.data_ptr()
        a.counter = ws.counter.data_ptr()
        if self.discrete_action:
            a.action_idx = noise.action_idx.data_ptr()
            a.action_out, a.one_hot = ws.action_out.data_ptr(), ws.one_hot.data_ptr()
        else:
            a.truncnorm = noise.truncnorm.data_ptr()
            a.lower, a.upper = ws.lower.data_ptr(), ws.upper.data_ptr()
            a.mean, a.var = ws.mean.data_ptr(), ws.var.data_ptr()
            a.elites = ws.elites.data_ptr()
            a.mean_hist, a.var_hist = ws.mean_hist.data_ptr(), ws.var_hist.data_ptr()
        a.dump = None if dump is None else _lib.ptr(dump, ws.device)
        return a

    @torch.no_grad()
    def plan(self, state, noise: Optional[CEMNoise] = None,
             dump: Optional[torch.Tensor] = None) -> CEMPlan:
        """One plan from `state` ([1, state_dim] FeatureData or tensor, on CUDA), launched on the
        current stream with no host synchronisation.  `noise` defaults to fresh draws from
        torch's CUDA generator.  `dump` (float32 [P, H, A + S + (2S + 1)G + 2], tests) receives
        iteration 0's per-step input and head outputs of every step a trajectory ran."""
        x = state.float_features if isinstance(state, rlt.FeatureData) else state
        if not x.is_cuda:
            raise _lib.Rb200Error(f"CEMPlannerNetwork: state is a {x.device} tensor; "
                                  "reagent_b200 runs on CUDA only (there is no CPU path)")
        if tuple(x.shape) != (1, self.state_dim):
            raise ValueError(f"CEMPlannerNetwork: state has shape {tuple(x.shape)}, expected "
                             f"{(1, self.state_dim)}")
        _lib.require_current_device(x.device)
        ws = self._workspace(x.device)
        if noise is None:
            noise = ws.noise.fill_()
        elif (noise.device != x.device or noise.discrete != self.discrete_action or
              (noise.iters, noise.P, noise.H, noise.A, noise.S, noise.num_models) !=
              (self.iters, self.cem_pop_size, self.plan_horizon_length, self.action_dim,
               self.state_dim, len(self.mem_net_list))):
            raise ValueError("CEMPlannerNetwork: the noise was made for another planner shape "
                             "or device (use new_noise)")
        ws.state.copy_(x.reshape(-1))
        ws.done.zero_()
        ws.n_iters.zero_()
        if not self.discrete_action:
            ws.mean.copy_(ws.mean0)
            ws.var.copy_(ws.var0)
        a = self._args(ws, noise, dump)
        lib, st = _lib.lib(), _lib.cur_stream()
        for i in range(self.iters):
            a.iter = i
            _lib.check(lib.rb200_cem_rollout(a, st), "rb200_cem_rollout")
        if self.discrete_action:
            return CEMPlan(action=ws.action_out, one_hot=ws.one_hot, values=ws.values,
                           elites=None, mean=None, var=None, n_iters=ws.n_iters)
        # the first action of the mean, from [lower, upper] to CONTINUOUS_TRAINING_ACTION_RANGE
        # (reagent/training/utils.py rescale_actions, in fp64)
        low, high = CONTINUOUS_TRAINING_ACTION_RANGE
        lo, hi = ws.orig_lower, ws.orig_upper
        action = ((ws.mean[:self.action_dim] - lo) / (hi - lo)) * (high - low) + low
        return CEMPlan(action=action, one_hot=None, values=ws.values, elites=ws.elites,
                       mean=ws.mean_hist, var=ws.var_hist, n_iters=ws.n_iters)

    @torch.no_grad()
    def forward(self, state: rlt.FeatureData):
        """The reference's outputs, on the CPU: (index, float32 one-hot [A]) for discrete
        actions, the float64 first action [A] for continuous ones."""
        p = self.plan(state)
        if self.discrete_action:
            return int(p.action.item()), p.one_hot.cpu()
        return p.action.cpu()
