"""The fused update shared by ReinforceTrainer and PPOTrainer: trajectories packed one after
another, one policy forward over all their rows, the value forwards, rb200_pg_returns,
rb200_pg_head, the backwards.  Launches of one update with a value net:

  rb200_mlp_forward x2   policy scores and V(state), activations saved
  rb200_mlp_forward      V(next_state)                 (PPO TD advantage with next_state)
  rb200_pg_returns       reward-to-go, whitening, clamp (skipped by the TD advantage)
  rb200_pg_head          advantage, policy and value losses, d loss / d scores, d loss / d V
  rb200_mlp_backward + rb200_mlp_wgrad, per network

then the value net's Adam step and the policy's.  A dueling policy adds its fold before the
forward and its unfold after the weight gradients.

Trajectory lengths change from update to update, so the workspace grows and never shrinks: the
kernels take the row count, and a shorter batch reuses the leading rows of every buffer.  The
weight-gradient partials are leading slices of a grow-only slab for the same reason."""
from typing import List

import torch

from .. import _lib
from ..core import types as rlt
from .workspace import NetWorkspace, Pins, batch_device, param_grads


def check_policy(trainer_name: str, policy, value_net) -> None:
    """The scorer must be a fused FullyConnectedDQN / DuelingQNetwork with one score per action,
    the sampler a SoftmaxActionSampler, the value net a fused network with one output."""
    from ..gym.policies import SoftmaxActionSampler
    from ..models import DuelingQNetwork, FullyConnectedDQN
    from ..models.fully_connected_network import FloatFeatureFullyConnected

    scorer = policy.scorer
    if not isinstance(scorer, (FullyConnectedDQN, DuelingQNetwork)) or scorer.num_atoms is not None:
        raise NotImplementedError(
            f"{trainer_name}: the policy's scorer must be a reagent_b200.models.FullyConnectedDQN "
            "or DuelingQNetwork without atoms (one score per action from the fused MLP kernel); "
            "got " + type(scorer).__name__)
    if scorer.action_dim > 1024:
        raise NotImplementedError(f"{trainer_name}: the loss head holds one row per warp: at most "
                                  "1024 actions")
    if not isinstance(policy.sampler, SoftmaxActionSampler):
        raise NotImplementedError(
            f"{trainer_name}: the policy's sampler must be a SoftmaxActionSampler (the loss head "
            "is its log-softmax); got " + type(policy.sampler).__name__)
    if value_net is not None and (not isinstance(value_net, FloatFeatureFullyConnected)
                                  or value_net.arena.dims[-1] != 1):
        raise NotImplementedError(
            f"{trainer_name}: value_net must be a reagent_b200 FloatFeatureFullyConnected with one "
            "output (e.g. net_builder.ValueFullyConnected); got " + type(value_net).__name__)


class PackedTrajectories:
    """The trajectories of one update on the GPU, one after another.  `offsets` [n + 1] (int32,
    device) is built from the tensor shapes and copied from pinned memory without waiting, so
    packing does not synchronise.  Every field is checked against the trajectory's length T,
    the policy's state width S and its action count A before anything is launched: the kernels
    take one row count for all of them.  log_prob is packed only when the loss reads it, and
    next_state / not_terminal only for the TD advantage (`td`)."""

    def __init__(self, trajs: List[rlt.PolicyGradientInput], pins: Pins, state_dim: int,
                 num_actions: int, *, log_prob: bool, td: bool):
        lengths = [_check_trajectory(k, t, state_dim, num_actions, log_prob, td)
                   for k, t in enumerate(trajs)]
        has_next = [t.next_state is not None for t in trajs]
        if td and any(has_next) and not all(has_next):
            raise ValueError("with the TD advantage either every trajectory of a minibatch has "
                             "next_state or none has")
        offs = [0]
        for n in lengths:
            offs.append(offs[-1] + n)
        self.lengths, self.rows, self.n_traj = lengths, offs[-1], len(trajs)
        dev = pins.device
        host = torch.tensor(offs, dtype=torch.int32).pin_memory()
        self.offsets = torch.empty(len(offs), dtype=torch.int32, device=dev)
        self.offsets.copy_(host, non_blocking=True)
        pins.keep += [host, self.offsets]

        def cat(ts):
            return pins.tensor(torch.cat([_lib.on_device(t.float(), dev) for t in ts]))

        self.state = cat([t.state.float_features for t in trajs])
        self.action = cat([t.action for t in trajs])
        self.reward = cat([t.reward for t in trajs])
        self.log_prob = cat([t.log_prob for t in trajs]) if log_prob else None
        self.mask = None
        if any(t.possible_actions_mask is not None for t in trajs):
            self.mask = cat([torch.ones(n, num_actions, device=dev) if t.possible_actions_mask is None
                             else t.possible_actions_mask for t, n in zip(trajs, lengths)])
        self.next_state = self.not_terminal = None
        if td:
            if all(has_next):
                self.next_state = cat([t.next_state.float_features for t in trajs])
            if any(t.not_terminal is not None for t in trajs):
                self.not_terminal = cat([_default_not_terminal(n, dev) if t.not_terminal is None
                                         else t.not_terminal for t, n in zip(trajs, lengths)])


def _check_trajectory(k: int, t: rlt.PolicyGradientInput, S: int, A: int, log_prob: bool,
                      td: bool) -> int:
    """The length T of trajectory k, after checking the shape of every field it uses."""
    def shape(x):
        return tuple(x.shape) if isinstance(x, torch.Tensor) else None

    def need(name, x, want):
        if shape(x) != want:
            raise ValueError(f"trajectory {k}: {name} has shape {shape(x)}, expected {want}")

    a = t.action
    if not isinstance(a, torch.Tensor) or a.ndim != 2 or a.shape[1] != A:
        raise ValueError(f"trajectory {k}: action has shape {shape(a)}, expected "
                         f"(T, {A}) one-hot rows")
    T = a.shape[0]
    if T == 0:
        raise ValueError(f"trajectory {k}: a trajectory must contain at least one step")
    need("state", t.state.float_features, (T, S))
    need("reward", t.reward, (T,))
    if log_prob:
        need("log_prob", t.log_prob, (T,))
    if t.possible_actions_mask is not None:
        need("possible_actions_mask", t.possible_actions_mask, (T, A))
    if td:
        if t.next_state is not None:
            need("next_state", t.next_state.float_features, (T, S))
        if t.not_terminal is not None:
            need("not_terminal", t.not_terminal, (T,))
    return T


def _default_not_terminal(n: int, device) -> torch.Tensor:
    nt = torch.ones(n, device=device)
    nt[-1] = 0.0
    return nt


class PolicyGradientStep:
    """Workspace and launches of the fused update of one trainer (policy, optional value net)."""

    def __init__(self, scorer, value_net):
        self.scorer = scorer
        self.value_net = value_net
        self.ws = None
        self._slabs = {}

    def workspace(self, rows: int, device):
        """Grow-only: new buffers only when `rows` exceeds every earlier update's row count."""
        ws = self.ws
        if ws is not None and ws["dev"] == device and ws["rows"] >= rows:
            return ws
        A = self.scorer.action_dim
        v = self.value_net
        nparts = 2 * (-(-rows // _lib.PG_ROWS_PER_BLOCK))
        self.ws = {
            "rows": rows, "dev": device,
            "policy": NetWorkspace(self.scorer.arena, rows, device),
            "scores": torch.empty(rows, A, device=device),
            "value": None if v is None else NetWorkspace(v.arena, rows, device),
            "v": None if v is None else torch.empty(rows, 1, device=device),
            "v_next": None if v is None else torch.empty(rows, 1, device=device),
            "returns": torch.empty(rows, device=device),
            "advantage": torch.empty(rows, device=device),
            "partials": torch.zeros(nparts, device=device),
            "loss": torch.zeros(2, device=device),
            "counter": torch.zeros(1, dtype=torch.int32, device=device),
        }
        return self.ws

    def _wgrad(self, arena, ws: NetWorkspace, x, rows: int):
        """rb200_mlp_wgrad into the leading `splits` rows of a grow-only partial slab."""
        lib = _lib.lib()
        splits = lib.rb200_wgrad_splits(rows)
        slab = self._slabs.get(id(arena))
        if slab is None or slab.shape[0] < splits or slab.device != arena.flat.device:
            # zeroed once: alignment padding is never written
            slab = self._slabs[id(arena)] = torch.zeros(splits, arena.n, device=arena.flat.device)
        arena.gpart = slab[:splits]
        rc = lib.rb200_mlp_wgrad(arena.desc(), x.data_ptr(), rows, ws.c, arena.gpart.data_ptr(),
                                 splits, _lib.cur_stream())
        _lib.check(rc, "rb200_mlp_wgrad")
        arena.grad_ready = True

    def returns_args(self, p: PackedTrajectories, ws, *, norm: int, offset_clamp_min: bool,
                     gamma: float, reward_clip: float, **_):
        """rb200_pg_returns' arguments for the packed batch `p` on workspace `ws`."""
        r = _lib.PgReturnsArgsT()
        r.n_traj, r.offsets, r.reward = p.n_traj, p.offsets.data_ptr(), p.reward.data_ptr()
        r.reward_clip, r.gamma = float(reward_clip), float(gamma)
        r.norm, r.offset_clamp_min = norm, int(bool(offset_clamp_min))
        r.returns = ws["returns"].data_ptr()
        return r

    def head_args(self, p: PackedTrajectories, ws, *, loss_kind: int, offset_clamp_min: bool,
                  td: bool, gamma: float, reward_clip: float, temperature: float,
                  value_scale: float, log_clip_param: float = 0.0, ppo_epsilon: float = 0.0,
                  entropy_weight: float = 0.0, do_backward: bool = True, **_):
        """rb200_pg_head's arguments for the packed batch `p` on workspace `ws`."""
        v = self.value_net
        a = _lib.PgHeadArgsT()
        a.rows, a.num_actions, a.n_traj = p.rows, self.scorer.action_dim, p.n_traj
        a.offsets = p.offsets.data_ptr()
        a.scores, a.mask, a.action = ws["scores"].data_ptr(), _lib.ptr(p.mask), p.action.data_ptr()
        a.logged_log_prob = _lib.ptr(p.log_prob)
        if td:
            a.advantage_kind = _lib.PG_ADV_TD
            a.reward = p.reward.data_ptr()
            a.next_value = ws["v_next"].data_ptr() if p.next_state is not None else None
            a.not_terminal = _lib.ptr(p.not_terminal)
            a.offset_clamp_min = int(bool(offset_clamp_min))
        else:
            a.advantage_kind = _lib.PG_ADV_RETURNS if v is None else _lib.PG_ADV_BASELINE
            a.returns = ws["returns"].data_ptr()
        a.value = None if v is None else ws["v"].data_ptr()
        a.temperature, a.gamma, a.reward_clip = float(temperature), float(gamma), float(reward_clip)
        a.log_clip_param, a.entropy_weight = float(log_clip_param), float(entropy_weight)
        # torch.clamp(rho, 1 - eps, 1 + eps) rounds the bounds from double
        a.ppo_clip_lo, a.ppo_clip_hi = 1.0 - ppo_epsilon, 1.0 + ppo_epsilon
        a.value_scale = float(value_scale)
        a.loss_kind = loss_kind
        a.advantage_out = ws["advantage"].data_ptr()
        a.dz = ws["policy"].dz[-1].data_ptr() if do_backward else None
        a.dz_value = ws["value"].dz[-1].data_ptr() if do_backward and v is not None else None
        a.loss_partials, a.loss = ws["partials"].data_ptr(), ws["loss"].data_ptr()
        a.tile_counter = ws["counter"].data_ptr()
        return a

    def run(self, p: PackedTrajectories, pins: Pins, *, td: bool, do_backward: bool = True, **kw):
        """Forwards, returns, head (and backwards into the gradient partials), with the settings
        `kw` of the trainer's `_settings`.  Returns the [2] device tensor (policy loss, value
        loss); no host synchronisation."""
        R = p.rows
        ws = self.workspace(R, pins.device)
        lib, st = _lib.lib(), _lib.cur_stream()
        ar = self.scorer.arena
        ar.refresh()  # no-op for plain MLPs; folds a dueling head
        ar.forward(p.state, ws["scores"][:R], save=ws["policy"] if do_backward else None)
        v = self.value_net
        if v is not None:
            v.arena.forward(p.state, ws["v"][:R], save=ws["value"] if do_backward else None)
            if td and p.next_state is not None:
                v.arena.forward(p.next_state, ws["v_next"][:R])
        if not td:
            _lib.check(lib.rb200_pg_returns(self.returns_args(p, ws, **kw), st), "rb200_pg_returns")
        a = self.head_args(p, ws, td=td, do_backward=do_backward, **kw)
        _lib.check(lib.rb200_pg_head(a, st), "rb200_pg_head")
        if do_backward:
            if v is not None:
                v.arena.backward(ws["value"], R)
                self._wgrad(v.arena, ws["value"], p.state, R)
            ar.backward(ws["policy"], R)
            self._wgrad(ar, ws["policy"], p.state, R)
            ar.finish_grads()  # dueling: folded-layer gradient -> true parameters
        return ws["loss"]

    def advantage(self, rows: int) -> torch.Tensor:
        """The advantages of the last update's rows (inspection / tests)."""
        return self.ws["advantage"][:rows]

    def returns(self, rows: int) -> torch.Tensor:
        return self.ws["returns"][:rows]


def pack(trajs: List[rlt.PolicyGradientInput], who: str, scorer, *, log_prob: bool, td: bool):
    """The trajectories packed for `scorer`, and the Pins that keep the packed tensors alive."""
    if not trajs:
        raise ValueError("an update needs at least one trajectory")
    pins = Pins(batch_device(trajs[0].state.float_features, who))
    return PackedTrajectories(trajs, pins, scorer.arena.dims[0], scorer.action_dim,
                              log_prob=log_prob, td=td), pins


def net_grads(net) -> List[torch.Tensor]:
    """Per-parameter gradients of the last fused backward of `net` (inspection / tests)."""
    return param_grads(net.arena, list(net.parameters()))
