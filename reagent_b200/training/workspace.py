"""Device workspaces for the fused trainers (activations, dZ, gradient partials) and the
marshalling every trainer does around the C entry points."""
import torch

from .. import _lib
from ..models.arena import ParamArena


class Pins:
    """The tensors of one C call: `pins(t)` makes `t` fp32, contiguous and resident on `device`,
    keeps that tensor alive in `keep` until the launch is enqueued and returns its device
    pointer (None -> NULL); `pins.tensor(t)` returns the tensor itself."""

    def __init__(self, device):
        self.device = device
        self.keep = []

    def tensor(self, t):
        if t is None:
            return None
        if t.dtype != torch.float32:
            t = t.float()
        t = _lib.on_device(t.contiguous(), self.device)
        self.keep.append(t)
        return t

    def __call__(self, t):
        return _lib.ptr(self.tensor(t), self.device)


def batch_device(state: torch.Tensor, who: str):
    """The device of a training batch (given its state features): a GPU, the current one."""
    if not state.is_cuda:
        raise _lib.Rb200Error(f"{who}: training batch must be on the GPU "
                              "(reagent_b200 has no CPU path)")
    _lib.require_current_device(state.device)
    return state.device


def discount_source(trainer, batch):
    """The per-row exponent of gamma -- the batch's time_diff with use_seq_num_diff_as_time_diff,
    its step with multi_steps -- or None for a constant gamma."""
    if trainer.use_seq_num_diff_as_time_diff:
        assert trainer.multi_steps is None
        return batch.time_diff.reshape(-1)
    if trainer.multi_steps is not None:
        assert batch.step is not None
        return batch.step.reshape(-1)
    return None


def loss_kind(q_network_loss: str) -> int:
    """The kernels' code of RLParameters.q_network_loss."""
    if q_network_loss == "mse":
        return _lib.LOSS_MSE
    if q_network_loss == "huber":
        return _lib.LOSS_HUBER
    raise Exception("Q-Network loss type {} not valid loss.".format(q_network_loss))


def register_reward_boosts(module, actions, reward_boost) -> None:
    """The [1, A] `reward_boosts` buffer of RLParameters.reward_boost ({action name: boost}) and
    `_has_reward_boost`, which tells the kernels whether to read it."""
    boosts = torch.zeros([1, len(actions)])
    module._has_reward_boost = False
    if reward_boost is not None:
        for k in reward_boost.keys():
            boosts[0, actions.index(k)] = reward_boost[k]
            module._has_reward_boost = True
    module.register_buffer("reward_boosts", boosts)


def ws_fits(ws, B: int, device) -> bool:
    """Whether a cached workspace dict was built for batch size B on `device`."""
    return ws is not None and ws["B"] == B and ws["dev"] == device


class NetWorkspace:
    """hidden[l] / dz[l] / input buffers of one network for a fixed batch size."""

    def __init__(self, arena: ParamArena, batch: int, device, need_input: bool = False):
        L = len(arena.acts)
        self.arena = arena
        self.batch = batch
        self.hidden = [torch.empty(batch, arena.dims[l + 1], device=device) for l in range(L - 1)]
        self.dz = [torch.empty(batch, arena.dims[l + 1], device=device) for l in range(L)]
        self.input = torch.empty(batch, arena.dims[0], device=device) if need_input else None
        self.c = _lib.NetWsT()
        for l, t in enumerate(self.hidden):
            self.c.hidden[l] = t.data_ptr()
        for l, t in enumerate(self.dz):
            self.c.dz[l] = t.data_ptr()
        self.c.input = None if self.input is None else self.input.data_ptr()


def check_sample_weight(w, batch: int):
    """Prioritized-replay importance weights of a distributional head: None or a [batch] float32
    tensor, with DQNTrainer's error for anything else."""
    if w is not None and (w.dtype != torch.float32 or w.shape != (batch,)):
        raise ValueError(f"importance_weights must be a [{batch}] float32 tensor, got "
                         f"{w.dtype} {tuple(w.shape)}")
    return w


def ensure_gpart(arena: ParamArena, splits: int):
    """[splits, n] gradient partial slab (zeroed once: alignment padding is never written)."""
    flat = arena.flat
    if arena.gpart is None or arena.gpart.shape[0] != splits or arena.gpart.device != flat.device:
        arena.gpart = torch.zeros(splits, arena.n, device=flat.device)
    return arena.gpart


def wgrad(arena: ParamArena, ws: NetWorkspace, net_input, batch: int):
    """Launch the split-K weight-gradient kernel for one network."""
    splits = _lib.lib().rb200_wgrad_splits(batch)
    g = ensure_gpart(arena, splits)
    rc = _lib.lib().rb200_mlp_wgrad(arena.desc(), _lib.ptr(net_input), batch, ws.c,
                                    g.data_ptr(), splits, _lib.cur_stream())
    _lib.check(rc, "rb200_mlp_wgrad")
    arena.grad_ready = True


def backward_wgrad(arena: ParamArena, ws: NetWorkspace, net_input, batch: int):
    """The whole backward of one network from the dZ of its last layer: dZ chain, then the
    weight gradients."""
    arena.backward(ws, batch)
    wgrad(arena, ws, net_input, batch)


def reduced_grad(arena: ParamArena) -> torch.Tensor:
    """Flat gradient = fixed-order sum of the partials (for inspection / all-reduce)."""
    assert arena.gpart is not None, "no gradient partials computed yet"
    out = torch.empty(arena.n, device=arena.flat.device)
    rc = _lib.lib().rb200_grad_reduce(arena.gpart.data_ptr(), arena.gpart.shape[0], arena.n,
                                      out.data_ptr(), _lib.cur_stream())
    _lib.check(rc, "rb200_grad_reduce")
    return out


def param_grads(arena: ParamArena, params):
    """Per-parameter gradient views (same shapes as the parameters)."""
    g = reduced_grad(arena)
    base = arena.flat.data_ptr()
    out = []
    for p in params:
        off = (p.data_ptr() - base) // 4
        out.append(g[off:off + p.numel()].view_as(p))
    return out
