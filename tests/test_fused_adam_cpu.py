"""FusedAdam's optimizer surface against torch.optim.Adam, without a GPU: constructor errors,
the state_dict layout, and checkpoints moving between the two optimizers in both directions."""
import pytest
import torch

from reagent_b200.models import FullyConnectedNetwork
from reagent_b200.optimizer import FusedAdam


def _net(seed=0):
    torch.manual_seed(seed)
    return FullyConnectedNetwork([5, 7, 3], ["relu", "linear"])


def _torch_adam_after_steps(net, steps=3, **kw):
    """A CPU torch.optim.Adam over `net`'s parameters with non-trivial state."""
    opt = torch.optim.Adam(net.parameters(), foreach=False, **kw)
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        for p in net.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    for p in net.parameters():
        p.grad = None
    return opt


def test_state_dict_layout_matches_torch_adam():
    net = _net()
    ref = _torch_adam_after_steps(_net(), lr=0.05, betas=(0.5, 0.9), eps=1e-3, weight_decay=1e-2)
    fused = FusedAdam(net.parameters(), lr=0.05, betas=(0.5, 0.9), eps=1e-3, weight_decay=1e-2)
    sd, rsd = fused.state_dict(), ref.state_dict()
    assert sd.keys() == rsd.keys()
    assert len(sd["param_groups"]) == len(rsd["param_groups"]) == 1
    assert sd["param_groups"][0].keys() == rsd["param_groups"][0].keys()
    for k in ("lr", "betas", "eps", "weight_decay", "params", "amsgrad", "maximize",
              "decoupled_weight_decay"):
        assert sd["param_groups"][0][k] == rsd["param_groups"][0][k], k
    assert sd["state"].keys() == rsd["state"].keys()
    for i in rsd["state"]:
        assert sd["state"][i].keys() == rsd["state"][i].keys()
        for k, v in rsd["state"][i].items():
            assert sd["state"][i][k].shape == v.shape, (i, k)
            assert sd["state"][i][k].dtype == v.dtype, (i, k)


def test_fused_adam_loads_torch_adam_state():
    src = _net()
    ref = _torch_adam_after_steps(src, steps=4, lr=0.05, betas=(0.5, 0.9), eps=1e-3,
                                  weight_decay=1e-2)
    fused = FusedAdam(_net(1).parameters())
    fused.load_state_dict(ref.state_dict())
    g = fused.param_groups[0]
    assert (g["lr"], tuple(g["betas"]), g["eps"], g["weight_decay"]) == (0.05, (0.5, 0.9), 1e-3, 1e-2)
    assert fused.num_steps == 4
    sd = fused.state_dict()
    for i, st in ref.state_dict()["state"].items():
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(sd["state"][i][k], st[k]), (i, k)
        assert float(sd["state"][i]["step"]) == float(st["step"])


def test_torch_adam_loads_fused_adam_state():
    src = _net()
    ref = _torch_adam_after_steps(src, steps=2, lr=0.05, betas=(0.5, 0.9), eps=1e-3)
    fused = FusedAdam(_net(1).parameters(), lr=0.05, betas=(0.5, 0.9), eps=1e-3)
    fused.load_state_dict(ref.state_dict())
    back = torch.optim.Adam(_net(2).parameters(), foreach=False)
    back.load_state_dict(fused.state_dict())
    for i, st in ref.state_dict()["state"].items():
        got = back.state_dict()["state"][i]
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(got[k], st[k]), (i, k)
    assert back.param_groups[0]["betas"] == (0.5, 0.9)
    assert back.param_groups[0]["amsgrad"] is False


@pytest.mark.parametrize("flag", ["amsgrad", "maximize", "decoupled_weight_decay"])
def test_load_state_dict_refuses_unsupported_torch_flags(flag):
    ref = _torch_adam_after_steps(_net(), steps=1)
    sd = ref.state_dict()
    sd["param_groups"][0][flag] = True
    fused = FusedAdam(_net(1).parameters(), lr=0.02)
    with pytest.raises(NotImplementedError, match=flag):
        fused.load_state_dict(sd)
    # nothing was loaded
    assert fused.param_groups[0]["lr"] == 0.02
    assert fused.num_steps == 0


@pytest.mark.parametrize("kw, exc", [
    (dict(amsgrad=True), NotImplementedError),
    (dict(maximize=True), NotImplementedError),
    (dict(lr=-1e-3), ValueError),
    (dict(eps=-1e-8), ValueError),
    (dict(betas=(1.0, 0.999)), ValueError),
    (dict(betas=(0.9, 1.0)), ValueError),
    (dict(betas=(-0.1, 0.999)), ValueError),
    (dict(betas=(0.9, -0.5)), ValueError),
])
def test_constructor_errors(kw, exc):
    with pytest.raises(exc):
        FusedAdam(_net().parameters(), **kw)


def test_constructor_accepts_boundary_values():
    opt = FusedAdam(_net().parameters(), lr=0.0, eps=0.0, betas=(0.0, 0.0))
    assert opt.param_groups[0]["betas"] == (0.0, 0.0)
