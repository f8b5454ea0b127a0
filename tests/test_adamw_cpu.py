"""AdamW / AMSGrad without a GPU: the oracle's restatement (oracle/adamw_oracle.py) against
torch.optim.AdamW and against golden vectors from the unmodified reference trainers
(oracle/make_adamw_golden.py); FusedAdamW's optimizer surface and checkpoints against
torch.optim.AdamW; the AdamW config; the Categorical net builder and the DiscreteC51DQN
manager; and the C ABI of the K3 arguments."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import td_oracle as O
from oracle.adamw_oracle import AdamWState
from reagent_b200.models import FullyConnectedNetwork
from reagent_b200.optimizer import FusedAdam, FusedAdamW
from tests import golden_util as G
from tests.golden_cases import _c51_kwargs, _dqn_kwargs, batch_at
from tests.golden_util import _cmp_losses, _cmp_net

ADAMW_CASES = ["qrdqn_adamw_amsgrad_cartpole", "c51_adamw_amsgrad_cartpole", "dqn_adamw_decay"]
SAC_ADAMW_CASES = ["sac_adamw_amsgrad"]


def _adamw_kw(meta):
    return dict(lr=meta["lr"], weight_decay=meta["weight_decay"], amsgrad=meta["amsgrad"])


# ---------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("weight_decay", [0.0, 0.01, 0.3])
def test_oracle_adamw_is_torch_adamw_bit_for_bit(amsgrad, weight_decay):
    g = torch.Generator().manual_seed(5)
    p0 = [torch.randn(7, 5, generator=g), torch.randn(3, generator=g)]
    ref = [torch.nn.Parameter(p.clone()) for p in p0]
    mine = [p.clone() for p in p0]
    kw = dict(lr=0.05, betas=(0.5, 0.9), eps=1e-3, weight_decay=weight_decay, amsgrad=amsgrad)
    topt = torch.optim.AdamW(ref, foreach=False, **kw)
    st = AdamWState(mine, **kw)
    for k in range(20):
        # shrinking gradients: exp_avg_sq falls, so the AMSGrad maximum is the one in use
        grads = [torch.randn(p.shape, generator=g) * 0.97 ** (3 * k) for p in p0]
        for p, gr in zip(ref, grads):
            p.grad = gr.clone()
        topt.step()
        st.step(mine, grads)
        for i, (a, b) in enumerate(zip(mine, ref)):
            assert torch.equal(a, b.detach()), (k, i)
            if amsgrad:
                assert torch.equal(st.vmax[i], topt.state[b]["max_exp_avg_sq"]), (k, i)
    if amsgrad:
        assert any(not torch.equal(st.vmax[i], st.v[i]) for i in range(2))


def _check_qnets(q, qt, arrays, tol):
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < tol and G.rel_err(ps[2 * i + 1], b) < tol, (prefix, i)


@pytest.mark.parametrize("name", ADAMW_CASES)
def test_adamw_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    opt = AdamWState(O.net_params(q), **_adamw_kw(meta))
    for it in range(meta["n_updates"]):
        batch = batch_at(arrays, it)
        if meta["kind"] == "qrdqn":
            loss = O.qrdqn_update(q, qt, opt, batch, gamma=meta["gamma"], tau=meta["tau"],
                                  num_atoms=meta["N"], double_q=meta["double_q"],
                                  maxq=meta["maxq"])[0]
        elif meta["kind"] == "c51":
            loss = O.c51_update(q, qt, opt, batch, gamma=meta["gamma"], tau=meta["tau"],
                                **_c51_kwargs(meta, batch))[0]
        else:
            loss = O.dqn_update(q, qt, opt, batch, gamma=meta["gamma"], tau=meta["tau"],
                                **_dqn_kwargs(meta, batch))[0]
        want = arrays["losses"][it]
        assert abs(loss - want) <= 1e-6 * max(1.0, abs(want)), (it, loss, want)
    _check_qnets(q, qt, arrays, 1e-6)


def sac_adamw_state(arrays, meta):
    """O.SacState of a golden SAC case with AdamWState on all four optimizers."""
    acts = meta["acts"] + ["linear"]
    st = O.SacState(G.oracle_net(arrays, "actor0", acts), G.oracle_net(arrays, "q1_0", acts),
                    G.oracle_net(arrays, "q2_0", acts), lr=meta["lr"],
                    entropy_temperature=meta["entropy_temperature"], learn_alpha=True,
                    target_entropy=meta["target_entropy"])
    kw = _adamw_kw(meta)
    st.adam_q1 = AdamWState(O.net_params(st.q1), **kw)
    st.adam_q2 = AdamWState(O.net_params(st.q2), **kw)
    st.adam_actor = AdamWState(O.net_params(st.actor), **kw)
    st.adam_alpha = AdamWState([st.log_alpha], **kw)
    return st


@pytest.mark.parametrize("name", SAC_ADAMW_CASES)
def test_sac_adamw_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    st = sac_adamw_state(arrays, meta)
    for it in range(meta["n_updates"]):
        out = O.sac_update(st, batch_at(arrays, it), torch.from_numpy(arrays[f"noise{it}.next"]),
                           torch.from_numpy(arrays[f"noise{it}.cur"]), gamma=meta["gamma"],
                           tau=meta["tau"])
        _cmp_losses(out["losses"], arrays["losses"][it], 2e-6)
    for prefix, net in (("actorN", st.actor), ("q1_N", st.q1), ("q1t_N", st.q1t),
                        ("q2_N", st.q2), ("q2t_N", st.q2t)):
        _cmp_net(net, arrays, prefix, 1e-5)
    assert G.rel_err(st.log_alpha, arrays["log_alpha_N"]) < 1e-6


# ---------------------------------------------------------------------------
# FusedAdamW's surface
# ---------------------------------------------------------------------------
def _net(seed=0):
    torch.manual_seed(seed)
    return FullyConnectedNetwork([5, 7, 3], ["relu", "linear"])


def _torch_adamw_after_steps(net, steps=3, **kw):
    opt = torch.optim.AdamW(net.parameters(), foreach=False, **kw)
    gen = torch.Generator().manual_seed(1)
    for k in range(steps):
        for p in net.parameters():
            p.grad = torch.randn(p.shape, generator=gen) * 0.5 ** k
        opt.step()
    for p in net.parameters():
        p.grad = None
    return opt


def test_fused_adamw_defaults_and_constructor_errors():
    opt = FusedAdamW(_net().parameters())
    ref = torch.optim.AdamW(_net().parameters())
    grp, rgrp = opt.param_groups[0], ref.param_groups[0]
    assert set(grp) == set(rgrp)
    for k in rgrp:
        if k != "params":
            assert grp[k] == rgrp[k], k
    assert grp["weight_decay"] == 0.01 and grp["decoupled_weight_decay"] is True
    assert opt.max_exp_avg_sq is None
    ams = FusedAdamW(_net().parameters(), amsgrad=True)
    assert ams.param_groups[0]["amsgrad"] is True
    assert ams.max_exp_avg_sq.shape == ams.exp_avg_sq.shape
    assert isinstance(ams, FusedAdam)
    with pytest.raises(NotImplementedError):
        FusedAdamW(_net().parameters(), maximize=True)
    for kw in (dict(lr=-1.0), dict(eps=-1.0), dict(betas=(1.0, 0.9)), dict(betas=(0.9, -0.1))):
        with pytest.raises(ValueError):
            FusedAdamW(_net().parameters(), **kw)
    # Adam keeps refusing amsgrad
    with pytest.raises(NotImplementedError):
        FusedAdam(_net().parameters(), amsgrad=True)


@pytest.mark.parametrize("amsgrad", [False, True])
def test_fused_adamw_state_dict_round_trip_with_torch_adamw(amsgrad):
    kw = dict(lr=0.05, betas=(0.5, 0.9), eps=1e-3, weight_decay=0.02, amsgrad=amsgrad)
    ref_net = _net()
    ref = _torch_adamw_after_steps(ref_net, **kw)
    fused = FusedAdamW(_net().parameters(), **kw)
    fused.load_state_dict(ref.state_dict())
    assert fused.num_steps == 3
    sd, rsd = fused.state_dict(), ref.state_dict()
    # the reference runs foreach=False on purpose; the fused optimizer reports torch's default
    assert ([dict(g, foreach=None) for g in sd["param_groups"]]
            == [dict(g, foreach=None) for g in rsd["param_groups"]])
    assert set(sd["state"]) == set(rsd["state"])
    for i, rst in rsd["state"].items():
        assert set(sd["state"][i]) == set(rst), i
        for k, v in rst.items():
            assert torch.equal(sd["state"][i][k], v), (i, k)
    back = torch.optim.AdamW(_net().parameters(), foreach=False, **kw)
    back.load_state_dict(sd)
    for i, rst in back.state_dict()["state"].items():
        for k, v in rst.items():
            assert torch.equal(v, rsd["state"][i][k]), (i, k)


def test_fused_adamw_refuses_states_it_does_not_implement():
    adam_state = torch.optim.Adam(_net().parameters()).state_dict()
    with pytest.raises(ValueError):
        FusedAdamW(_net().parameters()).load_state_dict(adam_state)
    ams_state = _torch_adamw_after_steps(_net(), amsgrad=True).state_dict()
    with pytest.raises(ValueError):
        FusedAdamW(_net().parameters()).load_state_dict(ams_state)
    plain_state = _torch_adamw_after_steps(_net()).state_dict()
    with pytest.raises(ValueError):
        FusedAdamW(_net().parameters(), amsgrad=True).load_state_dict(plain_state)
    max_state = torch.optim.AdamW(_net().parameters(), maximize=True).state_dict()
    with pytest.raises(NotImplementedError):
        FusedAdamW(_net().parameters()).load_state_dict(max_state)
    with pytest.raises(NotImplementedError):
        FusedAdam(_net().parameters()).load_state_dict(ams_state)


def test_adamw_config_in_the_optimizer_union():
    from reagent_b200.optimizer import Adam, AdamW, Optimizer__Union

    w = AdamW()
    assert (w.lr, w.betas, w.eps, w.weight_decay, w.amsgrad) == (1e-3, (0.9, 0.999), 1e-8, 0.01, False)
    u = Optimizer__Union(AdamW={"lr": 1e-3, "amsgrad": True})
    assert u.selected_field == "AdamW" and u.value == AdamW(amsgrad=True)
    opt = u.make_optimizer_scheduler(_net().parameters())["optimizer"]
    assert type(opt) is FusedAdamW
    g = opt.param_groups[0]
    assert (g["lr"], g["weight_decay"], g["amsgrad"], g["decoupled_weight_decay"]) == (1e-3, 0.01, True, True)
    d = Optimizer__Union.default().make_optimizer_scheduler(_net().parameters())["optimizer"]
    assert type(d) is FusedAdam and Optimizer__Union.default().value == Adam()
    with pytest.raises(NotImplementedError):
        Optimizer__Union(SGD={"lr": 0.1})


def test_trainers_take_adamw_through_their_optimizer_config():
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union, SoftUpdate
    from reagent_b200.training import C51Trainer

    dist = FullyConnectedDQN(4, 2, [8], ["relu"], num_atoms=5)
    q = CategoricalDQN(dist, qmin=0, qmax=4, num_atoms=5)
    t = C51Trainer(q, q.get_target_network(), actions=["0", "1"], num_atoms=5, qmin=0, qmax=4,
                   optimizer=Optimizer__Union(AdamW={"amsgrad": True}))
    assert [type(o) for o in t.optimizers()] == [FusedAdamW, SoftUpdate]
    assert t.optimizers()[0].amsgrad


# ---------------------------------------------------------------------------
# the Categorical builder and the DiscreteC51DQN manager
# ---------------------------------------------------------------------------
def test_categorical_builder_and_c51_manager():
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters as NP
    from reagent_b200.model_managers import DiscreteC51DQN
    from reagent_b200.models import CategoricalDQN
    from reagent_b200.net_builder import Categorical
    from reagent_b200.optimizer import Optimizer__Union

    s = NormalizationData({i: NP("CONTINUOUS", mean=0.0, stddev=1.0) for i in range(4)})
    b = Categorical()
    assert (b.sizes, b.activations) == ([256, 128], ["relu", "relu"])
    with pytest.raises(AssertionError):
        Categorical(sizes=[8], activations=["relu", "relu"])
    q = Categorical(sizes=[64, 64], activations=["leaky_relu"] * 2).build_q_network(s, 2, 21, 0, 40)
    assert isinstance(q, CategoricalDQN)
    assert q.distributional_network.fc.layers == [4, 64, 64, 42]
    assert torch.equal(q.support, torch.linspace(0, 40, 21))

    m = DiscreteC51DQN(actions=["0", "1"])
    assert (m.num_atoms, m.qmin, m.qmax, m.double_q_learning) == (51, -100, 200, True)
    assert isinstance(m.net_builder, Categorical)
    assert type(m.optimizer.value).__name__ == "Adam"
    DiscreteC51DQN(actions=["0", "1"], minibatch_size=512,
                   optimizer=Optimizer__Union(AdamW={"lr": 1e-3, "amsgrad": True}))
    with pytest.raises(AssertionError):
        DiscreteC51DQN(actions=["0"])
    with pytest.raises(AssertionError):
        DiscreteC51DQN(actions=["0", "1"], minibatch_size=100)
    with pytest.raises(RuntimeError):
        m.build_trainer({"state": s}, use_gpu=False)


# ---------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------
E_INVALID = -1  # RB200_E_INVALID, include/reagent_b200.h


def test_adam_soft_update_validates_the_new_fields():
    """Rejected on the host before any launch, so no device is needed."""
    from reagent_b200 import _lib

    lib = _lib.lib()
    buf = (C.c_float * 4)()
    step = (C.c_int64 * 1)()
    counter = (C.c_uint32 * 1)()
    p = C.cast(buf, C.c_void_p).value
    a = _lib.AdamArgsT()
    a.params = a.grad = a.exp_avg = a.exp_avg_sq = p
    a.step, a.block_counter = C.cast(step, C.c_void_p).value, C.cast(counter, C.c_void_p).value
    a.splits, a.n = 1, 4
    a.amsgrad = 1
    assert lib.rb200_adam_soft_update(a, None) == E_INVALID
    assert b"max_exp_avg_sq" in lib.rb200_last_error()
    a.amsgrad, a.decoupled_weight_decay = 0, 2
    assert lib.rb200_adam_soft_update(a, None) == E_INVALID
    assert b"0 or 1" in lib.rb200_last_error()
    a.decoupled_weight_decay, a.amsgrad = 0, -1
    assert lib.rb200_adam_soft_update(a, None) == E_INVALID
    assert np.isfinite(float(buf[0]))
