"""AdamW and AMSGrad on the fused K3 kernel (rb200_adam_soft_update / FusedAdamW):

* the kernel against torch.optim.AdamW(foreach=False) on the CPU, step by step, in each mode;
* FusedAdamW checkpoints moving through torch.optim.AdamW and back;
* the reference's trainers with AdamW (oracle/make_adamw_golden.py), through train_batch;
* the tensor-core weight images K3 writes for the DQN TD kernel;
* the captured online step of the QR-DQN and C51 managers at the CartPole configurations;
* the two-rank data-parallel update (skipped with fewer than two GPUs).
"""
import random

import numpy as np
import pytest
import torch

from reagent_b200 import _lib
from tests import golden_util as G
from tests.online_step import assert_captured_equals_eager, params, transition_stream
from tests.builders import _batch, _build_trainer, _free_port, _inject, _pbatch, _record, _rlt_batch
from tests.golden_cases import batch_at
from tests.kernel_util import BETAS, EPS, GRAD_SCALE, LR, NUM_SMS, TAU, _padded, _seq_sum

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _adamw_args(p_dev, parts_dev, m_dev, v_dev, vmax_dev, step, counter, weight_decay,
                amsgrad, tgt=None, exp_out=None):
    a = _lib.AdamArgsT()
    a.params, a.grad, a.splits, a.n = (p_dev.data_ptr(), parts_dev.data_ptr(), parts_dev.shape[0],
                                       p_dev.numel())
    a.exp_avg, a.exp_avg_sq = m_dev.data_ptr(), v_dev.data_ptr()
    a.step, a.block_counter = step.data_ptr(), counter.data_ptr()
    a.lr, a.beta1, a.beta2, a.eps, a.weight_decay = LR, BETAS[0], BETAS[1], EPS, weight_decay
    a.grad_scale = GRAD_SCALE
    if tgt is not None:
        a.target, a.tau, a.one_minus_tau = tgt.data_ptr(), TAU, float(1.0 - TAU)
    else:
        a.target, a.tau, a.one_minus_tau = None, 0.0, 1.0
    a.exp_out = None if exp_out is None else exp_out.data_ptr()
    a.dp_world = 1
    a.decoupled_weight_decay = 1
    a.amsgrad = int(amsgrad)
    a.max_exp_avg_sq = vmax_dev.data_ptr() if amsgrad else None
    return a


def _check_adamw_step(p_dev, m_dev, v_dev, vmax_dev, ref_p, opt, p_prev, v_prev, vmax_prev, g,
                      what):
    """One kernel step against torch.optim.AdamW's single-tensor CPU path from identical state,
    with the accounting of test_layer_kernels_gpu._check_adam_step: exp_avg equal; exp_avg_sq
    equal to the separately rounded rule and within 1 ulp of torch; the parameters equal to
    torch's rule run on the kernel's moments and the correctly rounded root, and equal to torch
    wherever both share a rounding path.  AMSGrad: max_exp_avg_sq is maximum(previous, the
    kernel's exp_avg_sq) bit for bit, and torch's own wherever the two exp_avg_sq agree.
    Afterwards torch's state is copied to the device, so the next step starts from identical
    state.  Returns (elements whose exp_avg_sq differs by 1 ulp, inexact CPU roots)."""
    st = opt.state[ref_p]
    grp = opt.param_groups[0]
    b2, wd, lr = grp["betas"][1], grp["weight_decay"], grp["lr"]
    assert torch.equal(m_dev.cpu(), st["exp_avg"]), (what, "exp_avg")
    v_got = v_dev.cpu()
    assert torch.equal(v_got, v_prev * b2 + ((1 - b2) * g) * g), (what, "exp_avg_sq rule")
    v_ulps = (v_got.view(torch.int32).long() - st["exp_avg_sq"].view(torch.int32).long()).abs()
    assert int(v_ulps.max()) <= 1, (what, "exp_avg_sq vs torch", int(v_ulps.max()))
    vd, vd_ref, same = v_got, st["exp_avg_sq"], v_ulps == 0
    if grp["amsgrad"]:
        vd, vd_ref = vmax_dev.cpu(), st["max_exp_avg_sq"]
        assert torch.equal(vd, torch.maximum(vmax_prev, v_got)), (what, "max_exp_avg_sq rule")
        same = vd.view(torch.int32) == vd_ref.view(torch.int32)
        assert torch.equal(vd[v_ulps == 0], vd_ref[v_ulps == 0]), (what, "max_exp_avg_sq vs torch")
    p_dec = p_prev * (1 - lr * wd) if wd != 0 else p_prev
    t = float(st["step"])
    step_size = lr / (1 - grp["betas"][0] ** t)
    bc2_sqrt = (1 - b2 ** t) ** 0.5
    cr = torch.from_numpy(np.sqrt(vd.numpy().astype(np.float64)).astype(np.float32))
    p_rule = p_dec + (-step_size * st["exp_avg"]) / (cr / bc2_sqrt + grp["eps"])
    p_got = p_dev.cpu()
    assert torch.equal(p_got, p_rule), (what, "params vs update rule", int((p_got != p_rule).sum()))
    inexact = vd_ref.sqrt() != torch.from_numpy(
        np.sqrt(vd_ref.numpy().astype(np.float64)).astype(np.float32))
    same_path = same & ~inexact
    assert torch.equal(p_got[same_path], ref_p.detach()[same_path]), (what, "params vs torch")
    v_dev.copy_(st["exp_avg_sq"])
    if grp["amsgrad"]:
        vmax_dev.copy_(st["max_exp_avg_sq"])
    p_dev.copy_(ref_p.detach())
    return int((v_ulps != 0).sum()), int(inexact.sum())


@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("splits", [1, 9, 64])
@pytest.mark.parametrize("n", [1, 255, 257, NUM_SMS * 4 * 256 + 3])
def test_adamw_soft_update_matches_torch_adamw(n, splits, weight_decay, amsgrad):
    lib = _lib.lib()
    g = torch.Generator().manual_seed(n * 131 + splits)
    p0 = torch.randn(n, generator=g)
    tgt0 = torch.randn(n, generator=g)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref_p], lr=LR, betas=BETAS, eps=EPS, weight_decay=weight_decay,
                            amsgrad=amsgrad, foreach=False)
    p_dev, tgt = p0.cuda(), tgt0.cuda()
    m_dev, v_dev = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    vmax_dev = torch.zeros(n, device="cuda")
    exp_out = _padded((n,))
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    v_off = inexact = 0
    for it in range(50):
        # gradients that shrink over the run: exp_avg_sq falls, and the AMSGrad maximum is used
        parts = torch.randn(splits, n, generator=g) * (0.1 * 0.95 ** it)
        parts_dev = parts.cuda()
        a = _adamw_args(p_dev, parts_dev, m_dev, v_dev, vmax_dev, step, counter, weight_decay,
                        amsgrad, tgt, exp_out)
        tgt_before = tgt.cpu()
        assert lib.rb200_adam_soft_update(a, _lib.cur_stream()) == 0, lib.rb200_last_error()
        torch.cuda.synchronize()
        p_prev = ref_p.detach().clone()
        st = opt.state.get(ref_p, {})
        v_prev = st["exp_avg_sq"].clone() if st else torch.zeros(n)
        vmax_prev = st["max_exp_avg_sq"].clone() if amsgrad and st else torch.zeros(n)
        ref_p.grad = _seq_sum(parts) * GRAD_SCALE
        g_eff = ref_p.grad.clone()
        opt.step()
        p_new = p_dev.cpu()
        assert torch.equal(tgt.cpu(), TAU * p_new + (1.0 - TAU) * tgt_before), (n, it, "target")
        e = exp_out.cpu()
        ulps = (e.view(torch.int32).long() - torch.exp(p_new).view(torch.int32).long()).abs()
        assert int(ulps.max()) <= 2, (n, it, "exp_out")
        dv, ds = _check_adamw_step(p_dev, m_dev, v_dev, vmax_dev, ref_p, opt, p_prev, v_prev,
                                   vmax_prev, g_eff, (n, splits, it))
        v_off, inexact = v_off + dv, inexact + ds
        assert int(step.item()) == it + 1
    if amsgrad and n > 1:
        assert not torch.equal(vmax_dev, v_dev), "the maximum never differed from exp_avg_sq"
    _record("adamw_vs_torch", n=n, splits=splits, weight_decay=weight_decay, amsgrad=amsgrad,
            steps=50, exp_avg_sq_1ulp_elements=v_off, inexact_sqrt_elements=inexact)


def test_amsgrad_nan_gradient_propagates_like_torch():
    """torch.maximum propagates NaN (fmaxf would drop it): a NaN gradient element leaves NaN in
    max_exp_avg_sq and the parameter for good, in both, and touches no other element."""
    lib = _lib.lib()
    n, splits = 257, 3
    g = torch.Generator().manual_seed(11)
    p0 = torch.randn(n, generator=g)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref_p], lr=LR, betas=BETAS, eps=EPS, amsgrad=True, foreach=False)
    p_dev = p0.cuda()
    m_dev, v_dev, vmax_dev = (torch.zeros(n, device="cuda") for _ in range(3))
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    bad = torch.tensor([0, 100, 256])
    for it in range(6):
        parts = torch.randn(splits, n, generator=g) * 0.1
        if it == 2:
            parts[1, bad] = float("nan")
        a = _adamw_args(p_dev, parts.cuda(), m_dev, v_dev, vmax_dev, step, counter, 1e-2, True)
        assert lib.rb200_adam_soft_update(a, _lib.cur_stream()) == 0, lib.rb200_last_error()
        ref_p.grad = _seq_sum(parts) * GRAD_SCALE
        opt.step()
        torch.cuda.synchronize()
        st = opt.state[ref_p]
        for got, want in ((vmax_dev, st["max_exp_avg_sq"]), (v_dev, st["exp_avg_sq"]),
                          (p_dev, ref_p.detach())):
            assert torch.equal(torch.isnan(got.cpu()), torch.isnan(want)), it
        if it >= 2:
            assert bool(torch.isnan(vmax_dev.cpu()[bad]).all())
            assert int(torch.isnan(vmax_dev).sum()) == len(bad)


def test_fused_adamw_state_dict_round_trip_with_torch_adamw():
    """10 FusedAdamW(amsgrad) steps; its state_dict resumes a CPU torch.optim.AdamW, and that
    one's state_dict resumes a fresh FusedAdamW.  Then 10 more steps on all three with the same
    gradients: the two FusedAdamWs stay bit-identical, and torch matches them step by step."""
    from reagent_b200.models import FullyConnectedNetwork
    from reagent_b200.optimizer import FusedAdamW

    torch.manual_seed(0)
    kw = dict(lr=LR, betas=BETAS, eps=EPS, weight_decay=1e-2, amsgrad=True)
    net = FullyConnectedNetwork([7, 33, 5], ["tanh", "linear"]).cuda()
    f1 = FusedAdamW(net.parameters(), **kw)
    ar = f1.arena
    g = torch.Generator().manual_seed(3)
    grads = [torch.randn(3, ar.n, generator=g) * (0.1 * 0.9 ** k) for k in range(20)]
    for k in range(10):
        f1.fused_step(grad=grads[k].cuda(), grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()

    cpu_net = FullyConnectedNetwork([7, 33, 5], ["tanh", "linear"])
    cpu_net.load_state_dict({k: v.cpu() for k, v in net.state_dict().items()})
    t2 = torch.optim.AdamW(cpu_net.parameters(), foreach=False, **kw)
    t2.load_state_dict(f1.state_dict())
    net3 = FullyConnectedNetwork([7, 33, 5], ["tanh", "linear"]).cuda()
    net3.load_state_dict(net.state_dict())
    f3 = FusedAdamW(net3.parameters(), amsgrad=True)
    f3.load_state_dict(t2.state_dict())
    assert f3.num_steps == 10 and f3.param_groups[0]["weight_decay"] == 1e-2

    params = list(cpu_net.parameters())
    v_off = inexact = 0
    for k in range(10, 20):
        gd = grads[k].cuda()
        f1.fused_step(grad=gd, grad_scale=GRAD_SCALE)
        f3.fused_step(grad=gd, grad_scale=GRAD_SCALE)
        flat_g = _seq_sum(grads[k]) * GRAD_SCALE
        prev = [p.detach().clone() for p in params]
        for l in range(2):
            params[2 * l].grad = ar.weight_view(flat_g, l).clone()
            params[2 * l + 1].grad = ar.bias_view(flat_g, l).clone()
        before = [(t2.state[p]["exp_avg_sq"].clone(), t2.state[p]["max_exp_avg_sq"].clone(),
                   p.grad.clone()) for p in params]
        t2.step()
        torch.cuda.synchronize()
        for l in range(2):
            for j, view in enumerate((ar.weight_view, ar.bias_view)):
                # the arena's alignment padding is not state: compare the parameters only
                for a1, a3 in ((f1.arena.flat, f3.arena.flat), (f1.exp_avg, f3.exp_avg),
                               (f1.exp_avg_sq, f3.exp_avg_sq),
                               (f1.max_exp_avg_sq, f3.max_exp_avg_sq)):
                    assert torch.equal(view(a1, l), view(a3, l)), (k, l, j)
                i = 2 * l + j
                dv, ds = _check_adamw_step(view(f1.arena.flat, l), view(f1.exp_avg, l),
                                           view(f1.exp_avg_sq, l), view(f1.max_exp_avg_sq, l),
                                           params[i], t2, prev[i], *before[i],
                                           ("round trip", k, l, j))
                v_off, inexact = v_off + dv, inexact + ds
        # keep f3 on the same (torch-synchronised) state as f1
        f3.arena.flat.copy_(f1.arena.flat)
        f3.exp_avg_sq.copy_(f1.exp_avg_sq)
        f3.max_exp_avg_sq.copy_(f1.max_exp_avg_sq)
    assert f1.num_steps == f3.num_steps == 20
    _record("adamw_state_dict_round_trip", exp_avg_sq_1ulp_elements=v_off,
            inexact_sqrt_elements=inexact)


# ---------------------------------------------------------------------------
# the reference's trainers with AdamW
# ---------------------------------------------------------------------------
def _adamw_close(w_gpu, w_ref, meta, what):
    """Post-update parameters: Adam turns gradient elements within fp32 noise of zero into
    +-lr moves, so every element is bounded by the step budget (n_updates * 2 * lr) widened by
    the decay (n_updates * lr * wd * |p|), and the typical element lies within 2 % of a step."""
    w_ref = torch.as_tensor(w_ref, dtype=torch.float64)
    d = (w_gpu.detach().cpu().double() - w_ref).abs()
    k, lr, wd = meta["n_updates"], meta["lr"], meta["weight_decay"]
    bound = k * (2 * lr + lr * wd * w_ref.abs()) * 1.01
    assert bool((d <= bound).all()), (what, float((d - bound).max()))
    assert float(d.median()) < 0.02 * lr, (what, float(d.median()))


def _union(meta):
    from reagent_b200.optimizer import Optimizer__Union

    return Optimizer__Union(AdamW={"lr": meta["lr"], "weight_decay": meta["weight_decay"],
                                   "amsgrad": meta["amsgrad"]})


def _discrete_trainer(meta, arrays):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import CategoricalDQN, DuelingQNetwork, FullyConnectedDQN
    from reagent_b200.training import C51Trainer, DQNTrainer, QRDQNTrainer

    S, A = meta["S"], meta["A"]
    actions = [str(i) for i in range(A)]
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"], maxq_learning=True,
                      q_network_loss=meta.get("loss", "mse"))
    ev = EvaluationParameters(calc_cpe_in_training=False)
    if meta["kind"] == "qrdqn":
        q = DuelingQNetwork.make_fully_connected(S, A, meta["sizes"], meta["acts"], num_atoms=meta["N"])
        qt = q.get_target_network()
        G.load_into_module(arrays, "q0", q)
        G.load_into_module(arrays, "qt0", qt)
        t = QRDQNTrainer(q, qt, actions=actions, rl=rl, double_q_learning=True,
                         num_atoms=meta["N"], minibatch_size=meta["B"], optimizer=_union(meta),
                         evaluation=ev)
        return t.cuda(), (q, qt)
    if meta["kind"] == "c51":
        dist = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"], num_atoms=meta["N"])
        G.load_into_module(arrays, "q0", dist)
        q = CategoricalDQN(dist, qmin=meta["qmin"], qmax=meta["qmax"], num_atoms=meta["N"])
        qt = q.get_target_network()
        G.load_into_module(arrays, "qt0", qt.distributional_network)
        t = C51Trainer(q.cuda(), qt.cuda(), actions=actions, rl=rl, double_q_learning=True,
                       minibatch_size=meta["B"], num_atoms=meta["N"], qmin=meta["qmin"],
                       qmax=meta["qmax"], optimizer=_union(meta))
        return t.cuda(), (q.distributional_network, qt.distributional_network)
    q = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"])
    qt = q.get_target_network()
    G.load_into_module(arrays, "q0", q)
    G.load_into_module(arrays, "qt0", qt)
    t = DQNTrainer(q, qt, actions=actions, rl=rl, double_q_learning=True,
                   minibatch_size=meta["B"], optimizer=_union(meta), evaluation=ev)
    return t.cuda(), (q, qt)


@pytest.mark.parametrize("name", ["qrdqn_adamw_amsgrad_cartpole", "c51_adamw_amsgrad_cartpole",
                                  "dqn_adamw_decay"])
def test_discrete_trainers_with_adamw_match_reference(name):
    from reagent_b200.optimizer import FusedAdamW

    arrays, meta = G.load(name)
    t, (q, qt) = _discrete_trainer(meta, arrays)
    assert type(t.optimizers()[0]) is FusedAdamW
    assert t.optimizers()[0].amsgrad == meta["amsgrad"]
    for it in range(meta["n_updates"]):
        loss = float(t.train_batch(_batch(batch_at(arrays, it, "cuda"), meta), it))
        want = arrays["losses"][it]
        assert abs(loss - want) <= TOL * max(1.0, abs(want)), (it, loss, want)
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = list(net.parameters())
        pairs = G.net_pairs(arrays, prefix)
        assert len(ps) == 2 * len(pairs)
        for i, (w, b) in enumerate(pairs):
            _adamw_close(ps[2 * i], w, meta, (prefix, "W", i))
            _adamw_close(ps[2 * i + 1], b, meta, (prefix, "b", i))


def test_sac_with_adamw_amsgrad_matches_reference():
    """AdamW + AMSGrad on all four optimizers, log_alpha's ScalarArena and exp_out included."""
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.optimizer import FusedAdamW
    from reagent_b200.training import SACTrainer

    arrays, meta = G.load("sac_adamw_amsgrad")
    S, A = meta["S"], meta["A"]
    actor = GaussianFullyConnectedActor(S, A, meta["sizes"], meta["acts"])
    q1 = FullyConnectedCritic(S, A, meta["sizes"], meta["acts"])
    q2 = FullyConnectedCritic(S, A, meta["sizes"], meta["acts"])
    for m, prefix in ((actor, "actor0"), (q1, "q1_0"), (q2, "q2_0")):
        G.load_into_module(arrays, prefix, m)
    t = SACTrainer(actor, q1, q2, rl=RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"]),
                   q_network_optimizer=_union(meta), actor_network_optimizer=_union(meta),
                   alpha_optimizer=_union(meta), minibatch_size=meta["B"],
                   entropy_temperature=meta["entropy_temperature"],
                   target_entropy=meta["target_entropy"]).cuda()
    opts = t.optimizers()
    assert [type(o) for o in opts[:4]] == [FusedAdamW] * 4 and all(o.amsgrad for o in opts[:4])
    for it in range(meta["n_updates"]):
        _inject(t, arrays, it)
        closs, aloss = t.train_batch(_pbatch(batch_at(arrays, it, "cuda")), it)
        ref = arrays["losses"][it]
        assert abs(float(closs[0]) - ref[0]) <= 2e-5 * max(1.0, abs(ref[0])), (it, float(closs[0]), ref[0])
    for mod, prefix in ((t.actor_network, "actorN"), (t.q1_network, "q1_N"),
                        (t.q1_network_target, "q1t_N"), (t.q2_network, "q2_N"),
                        (t.q2_network_target, "q2t_N")):
        for i, seq in enumerate(mod.fc.dnn):
            _adamw_close(seq[0].weight, arrays[f"{prefix}.W{i}"], meta, (prefix, "W", i))
            _adamw_close(seq[0].bias, arrays[f"{prefix}.b{i}"], meta, (prefix, "b", i))
    _adamw_close(t.log_alpha.reshape(-1), arrays["log_alpha_N"].reshape(-1), meta, "log_alpha")
    # exp_out: the entropy temperature K3 writes is exp of the updated log_alpha
    alpha = float(t.entropy_temperature) if not torch.is_tensor(t.entropy_temperature) \
        else float(t.entropy_temperature.reshape(-1)[0])
    assert abs(alpha - float(torch.exp(t.log_alpha.detach().reshape(-1)[0].cpu()))) <= 1e-6 * alpha


@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("S,sizes,A", [(128, [256, 128], 16), (36, [300, 130, 20], 9)])
def test_adamw_writes_the_same_weight_images_as_the_pack_kernel(S, sizes, A, amsgrad):
    from reagent_b200.optimizer import Optimizer__Union, FusedAdamW

    B = 64
    meta = dict(S=S, A=A, B=B, sizes=sizes, acts=["relu"] * len(sizes), gamma=0.9, tau=0.1,
                loss="huber", maxq=True, multi_steps=None, time_diff=False, boost=None,
                double_q=True, lr=1e-2, n_updates=1)
    torch.manual_seed(S)
    t = _build_trainer(meta)
    t.q_network_optimizer = Optimizer__Union(AdamW={"lr": 1e-2, "amsgrad": amsgrad})
    t._optimizers_cache = None
    assert type(t.optimizers()[0]) is FusedAdamW
    act = torch.randint(A, (B,))
    nt = (torch.rand(B, 1) > 0.1).float()
    b = dict(state=torch.randn(B, S), next_state=torch.randn(B, S), reward=torch.randn(B, 1),
             time_diff=torch.ones(B, 1), step=None, not_terminal=nt,
             action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    batch = _rlt_batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    for _ in range(3):
        t.train_batch(batch)
    assert t._tc_images_current(), "the AdamW step should have refreshed the images"
    pack = t._last_td_call[-1]
    assert pack is not None
    torch.cuda.synchronize()
    by_adam = pack.clone()
    fresh = torch.zeros_like(pack)
    rc = _lib.lib().rb200_dqn_tc_pack(t.q_network.arena.desc(), t.q_network_target.arena.desc(), 1, 1,
                                      fresh.data_ptr(), fresh.numel(), _lib.cur_stream())
    _lib.check(rc, "rb200_dqn_tc_pack")
    torch.cuda.synchronize()
    assert torch.equal(by_adam, fresh)


# ---------------------------------------------------------------------------
# the captured online step of the managers at the CartPole configurations
# ---------------------------------------------------------------------------
def _cartpole_trainer(kind):
    """reagent/gym/tests/configs/cartpole/discrete_{qr,c51}_cartpole_online.yaml"""
    from reagent_b200.core.parameters import (NormalizationData, NormalizationKey,
                                              NormalizationParameters as NP, RLParameters)
    from reagent_b200.model_managers import DiscreteC51DQN, DiscreteQRDQN
    from reagent_b200.net_builder import Categorical, DuelingQuantile
    from reagent_b200.optimizer import Optimizer__Union

    rl = RLParameters(gamma=0.9, target_update_rate=0.05, maxq_learning=True, temperature=1.0)
    opt = Optimizer__Union(AdamW={"lr": 0.001, "amsgrad": True})
    acts = dict(sizes=[64, 64], activations=["leaky_relu", "leaky_relu"])
    if kind == "qrdqn":
        m = DiscreteQRDQN(actions=["0", "1"], rl=rl, double_q_learning=True, num_atoms=11,
                          minibatch_size=512, optimizer=opt, net_builder=DuelingQuantile(**acts))
    else:
        m = DiscreteC51DQN(actions=["0", "1"], rl=rl, double_q_learning=True, num_atoms=21,
                           qmin=0, qmax=40, minibatch_size=512, optimizer=opt,
                           net_builder=Categorical(**acts))
    s = NormalizationData({i: NP("CONTINUOUS", mean=0.0, stddev=1.0) for i in range(4)})
    torch.manual_seed(4)
    return m.build_trainer({NormalizationKey.STATE: s}, use_gpu=True), m.minibatch_size


@pytest.mark.parametrize("with_per", [False, True])
@pytest.mark.parametrize("kind", ["qrdqn", "c51"])
def test_cartpole_online_step_with_adamw_captured_equals_eager(kind, with_per):
    """30 online steps (one transition added per step) through graph replay and through eager
    launches of the same update: losses and parameters agree bit for bit."""
    from reagent_b200.optimizer import FusedAdamW
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    n_steps = 30
    base = transition_stream(3000, 7, 4, 2)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=10, eps=1e-6) if with_per else None

    def setup():
        t, B = _cartpole_trainer(kind)
        assert type(t.optimizers()[0]) is FusedAdamW and t.optimizers()[0].amsgrad
        rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=4096, batch_size=B)
        rb.add_batch(**base)
        random.seed(5)
        return FusedDqnStep(t, rb, B, rng="device", online=True, per=per), None

    assert_captured_equals_eager(
        setup, transition_stream(n_steps, 8, 4, 2), n_steps,
        lambda f: [params(f.trainer.q_network), params(f.trainer.q_network_target),
                   f.trainer.optimizers()[0].max_exp_avg_sq.clone()],
        drop_priority=(lambda i: i % 2) if with_per else None)


# ---------------------------------------------------------------------------
# data parallel
# ---------------------------------------------------------------------------
def _dp_worker(rank, world, port, use_p2p, out):
    import os

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        import bench
        from reagent_b200.core import types as rlt
        from reagent_b200.optimizer import Optimizer__Union
        from reagent_b200.training.data_parallel import enable_p2p, shard_rows

        if use_p2p:
            enable_p2p(dist.group.WORLD)
        cfg = dict(bench.CONFIGS[2], B=1024)
        B, S, A = cfg["B"], cfg["S"], cfg["A"]
        lo, hi = shard_rows(B, rank, world)
        g = torch.Generator(device=dev).manual_seed(3)
        r = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
        state, nstate, reward = r(B, S), r(B, S), r(B, 1)
        nt = (torch.rand(B, 1, device=dev, generator=g) > 0.05).float()
        act = torch.nn.functional.one_hot(torch.randint(A, (B,), device=dev, generator=g), A).float()

        def mk(sl):
            return rlt.DiscreteDqnInput(
                state=rlt.FeatureData(state[sl]), next_state=rlt.FeatureData(nstate[sl]),
                reward=reward[sl], time_diff=None, step=None, not_terminal=nt[sl],
                action=act[sl], next_action=act[sl] * nt[sl],
                possible_actions_mask=torch.ones(B, A, device=dev)[sl],
                possible_next_actions_mask=torch.ones(B, A, device=dev)[sl], extras=rlt.ExtraData())

        ts = []
        for _ in range(2):
            t = bench.build_trainer(cfg, dev, seed=11)
            t.q_network_optimizer = Optimizer__Union(AdamW={"lr": bench.LR, "amsgrad": True})
            t._optimizers_cache = None
            ts.append(t)
        t_dp, t_full = ts
        for it in range(2):  # two updates: the second uses the other buffer parity
            t_full.train_batch(mk(slice(0, B)), it)
            t_dp.train_batch(mk(slice(lo, hi)), it, process_group=dist.group.WORLD)
        torch.cuda.synchronize()
        worst = frac = 0.0
        for a, b in zip(t_dp.parameters(), t_full.parameters()):
            scale = float(b.abs().max()) + 1e-30
            d = (a.detach().double() - b.detach().double()).abs()
            worst = max(worst, float(d.max()) / scale)
            frac = max(frac, float((d > 1e-5 * scale).double().mean()))
        flat = torch.cat([p.detach().reshape(-1) for p in t_dp.parameters()])
        flat = torch.cat([flat, t_dp.optimizers()[0].max_exp_avg_sq])
        other = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(other, flat)
        out.put((rank, worst, frac, all(torch.equal(o, flat) for o in other)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_p2p", [True, False])
def test_two_rank_adamw_amsgrad_update_matches_full_batch(use_p2p):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp


    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, use_p2p, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(500)
        assert p.exitcode == 0, f"worker exit code {p.exitcode}"
    for rank, worst, frac, same in (out.get(timeout=10) for _ in range(2)):
        assert worst < 0.05, (rank, worst)
        assert frac < 2e-3, (rank, frac)
        assert same, "ranks diverged"
