"""GPU parity of the fused SAC / TD3 updates vs golden vectors from the unmodified
reference trainers (noise draws injected) and vs the CPU oracle at BASELINE config sizes.
Tolerance 1e-5 relative fp32 (north star); SAC's actor gradients pass through
atanh(tanh(x)), whose fp32 round trip is ill-conditioned near saturation, and get 5e-5."""
import numpy as np
import pytest
import torch

from oracle import td_oracle as O
from tests import golden_util as G
from tests.builders import _build_sac, _build_td3, _inject, _net_arrays, _pbatch, _rand_net
from tests.golden_cases import SAC_CASES, TD3_CASES
from tests.golden_util import TOL, _adam_close, _cmp_module

pytestmark = pytest.mark.gpu


def _check_sac_final(t, arrays, meta):
    _cmp_module(t.actor_network, arrays, "actorN", 2e-5)
    _cmp_module(t.q1_network, arrays, "q1_N")
    _cmp_module(t.q1_network_target, arrays, "q1t_N")
    if meta["twin"]:
        _cmp_module(t.q2_network, arrays, "q2_N")
        _cmp_module(t.q2_network_target, arrays, "q2t_N")
    if meta["learn_alpha"]:
        assert G.rel_err(t.log_alpha, arrays["log_alpha_N"]) < TOL


@pytest.mark.parametrize("name", SAC_CASES)
def test_sac_generator_path_matches_reference(name):
    from reagent_b200.training import run_update

    arrays, meta = G.load(name)
    t = _build_sac(meta, arrays)
    batch = _pbatch(G.batch_tensors(arrays, "cuda"))
    for it in range(meta["n_updates"]):
        _inject(t, arrays, it)
        if it == 0:
            opts = t.optimizers()
            nets = [t.q1_network] + ([t.q2_network] if meta["twin"] else []) + [t.actor_network]
            for oi, opt in enumerate(opts):
                loss = t.training_step(batch, it, oi)
                if oi < len(nets):
                    tol = 5e-5 if nets[oi] is t.actor_network else TOL
                    for pi, g in enumerate(t.net_grads(nets[oi])):
                        assert G.rel_err(g, arrays[f"grad0.opt{oi}.{pi}"]) < tol, (oi, pi)
                elif meta["learn_alpha"] and oi == len(nets):
                    assert G.rel_err(t._ws["alpha_grad"], arrays[f"grad0.opt{oi}.0"]) < TOL
                if oi < len(opts) - 1:
                    ref = arrays["losses"][it][oi]
                    assert abs(float(loss.detach()) - ref) <= TOL * max(1.0, abs(ref)), (oi, float(loss.detach()), ref)
                opt.zero_grad()
                loss.backward()
                opt.step()
        else:
            losses = run_update(t, batch, it)
            for oi, ref in enumerate(arrays["losses"][it]):
                assert abs(float(losses[oi].detach()) - ref) <= 2e-5 * max(1.0, abs(ref)), (it, oi)
    _check_sac_final(t, arrays, meta)


@pytest.mark.parametrize("name", SAC_CASES)
def test_sac_fast_path_matches_reference(name):
    arrays, meta = G.load(name)
    t = _build_sac(meta, arrays)
    batch = _pbatch(G.batch_tensors(arrays, "cuda"))
    for it in range(meta["n_updates"]):
        _inject(t, arrays, it)
        closs, aloss = t.train_batch(batch, it)
        ref = arrays["losses"][it]
        assert abs(float(closs[0]) - ref[0]) <= 2e-5 * max(1.0, abs(ref[0]))
    _check_sac_final(t, arrays, meta)


def _check_td3_final(t, arrays, meta):
    _cmp_module(t.actor_network, arrays, "actorN")
    _cmp_module(t.actor_network_target, arrays, "actort_N")
    _cmp_module(t.q1_network, arrays, "q1_N")
    _cmp_module(t.q1_network_target, arrays, "q1t_N")
    if meta["twin"]:
        _cmp_module(t.q2_network, arrays, "q2_N")
        _cmp_module(t.q2_network_target, arrays, "q2t_N")


@pytest.mark.parametrize("name", TD3_CASES)
@pytest.mark.parametrize("fast", [False, True])
def test_td3_matches_reference(name, fast):
    from reagent_b200.training import run_update

    arrays, meta = G.load(name)
    t = _build_td3(meta, arrays)
    batch = _pbatch(G.batch_tensors(arrays, "cuda"))
    for it in range(meta["n_updates"]):
        _inject(t, arrays, it)
        ref = arrays["losses"][it]
        if fast:
            closs, aloss = t.train_batch(batch, it)
            assert abs(float(closs[0]) - ref[0]) <= TOL * max(1.0, abs(ref[0]))
            assert (aloss is None) == bool(np.isnan(ref[-1]))
        else:
            if it == 0:
                opts = t.optimizers()
                nets = [t.q1_network] + ([t.q2_network] if meta["twin"] else []) + [t.actor_network]
                for oi, opt in enumerate(opts):
                    loss = t.training_step(batch, it, oi)
                    if oi < len(nets):
                        for pi, g in enumerate(t.net_grads(nets[oi])):
                            assert G.rel_err(g, arrays[f"grad0.opt{oi}.{pi}"]) < TOL, (oi, pi)
                    opt.zero_grad()
                    loss.backward()
                    opt.step()
            else:
                losses = run_update(t, batch, it)
                for oi, r in enumerate(ref):
                    if np.isnan(r):
                        assert losses[oi] is None
                    else:
                        assert abs(float(losses[oi].detach()) - r) <= TOL * max(1.0, abs(r))
    _check_td3_final(t, arrays, meta)


def test_sac_config4_shard_matches_oracle():
    """BASELINE config 4 per-GPU shard: S=256, A=32, B=2048, [256,256] nets, twin critics."""
    S, A, B = 256, 32, 2048
    meta = dict(S=S, A=A, B=B, sizes=[256, 256], acts=["relu", "relu"], twin=True,
                learn_alpha=True, gamma=0.99, tau=0.005, lr=1e-3, entropy_temperature=0.1,
                target_entropy=-float(A), backprop=True, n_updates=2)
    gen = torch.Generator().manual_seed(0)
    actor = _rand_net([S, 256, 256, 2 * A], ["relu", "relu", "linear"], gen)
    q1 = _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen)
    q2 = _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen)
    arrays = {}
    _net_arrays(arrays, "actor0", actor)
    _net_arrays(arrays, "q1_0", q1)
    _net_arrays(arrays, "q2_0", q2)
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             action=torch.rand(B, A, generator=gen) * 1.98 - 0.99,
             next_action=torch.zeros(B, A), reward=torch.randn(B, 1, generator=gen),
             not_terminal=(torch.rand(B, 1, generator=gen) > 0.005).float())
    t = _build_sac(meta, arrays)
    st = O.SacState(actor, q1, q2, lr=1e-3, entropy_temperature=0.1, learn_alpha=True,
                    target_entropy=-float(A))
    gb = _pbatch({k: v.cuda() for k, v in b.items()})
    for it in range(meta["n_updates"]):
        nn_, nc = torch.randn(B, A, generator=gen), torch.randn(B, A, generator=gen)
        arrays[f"noise{it}.next"], arrays[f"noise{it}.cur"] = nn_.numpy(), nc.numpy()
        _inject(t, arrays, it)
        out = O.sac_update(st, b, nn_, nc, gamma=0.99, tau=0.005)
        if it == 0:
            # gradients straight out of the fused backward (before Adam touches them)
            t._critic_step(gb, t.actor_network, t.q1_network_target, t.q2_network_target,
                           t._fill_critic)
            for pi, g in enumerate(t.net_grads(t.q1_network)):
                G.grad_close(g, out["grads"]["q1"][pi], ("q1 grad", pi))
            for pi, g in enumerate(t.net_grads(t.q2_network)):
                G.grad_close(g, out["grads"]["q2"][pi], ("q2 grad", pi))
            # the entropy term passes through atanh(tanh(x)) (ill-conditioned near saturation,
            # reagent/models/actor.py:243-251): 5e-5 on the target instead of 1e-5
            assert G.rel_err(t._ws["td_target"], out["target"].reshape(-1)) < 5e-5
        closs, aloss = t.train_batch(gb, it)
        assert abs(float(closs[0]) - out["losses"][0]) <= 2e-5 * max(1.0, abs(out["losses"][0]))
        assert abs(float(closs[1]) - out["losses"][1]) <= 2e-5 * max(1.0, abs(out["losses"][1]))
        assert abs(float(aloss[0]) - out["losses"][2]) <= 2e-5 * max(1.0, abs(out["losses"][2]))
    # Post-Adam weights: Adam moves an element by ~lr*g/(|g|+eps) per step, so an element whose
    # gradient is within fp32 noise of zero can move by up to lr in EITHER direction however
    # well the gradients agree (they agree to 1e-5 above).  Hence: hard bound n*2*lr on every
    # element, and all but a vanishing fraction of elements within 1e-5 of the weight scale.
    for net, onet in ((t.q1_network, st.q1), (t.actor_network, st.actor)):
        for i, seq in enumerate(net.fc.dnn):
            _adam_close(seq[0].weight, onet["W"][i], meta)
    assert G.rel_err(t.log_alpha, st.log_alpha) < TOL


def test_td3_config5_shard_matches_oracle():
    """BASELINE config 5 per-GPU shard: S=512, A=64, B=2048, [256,256] nets, twin critics."""
    S, A, B = 512, 64, 2048
    meta = dict(S=S, A=A, B=B, sizes=[256, 256], acts=["relu", "relu"], twin=True, gamma=0.99,
                tau=0.005, lr=1e-3, noise_variance=0.2, noise_clip=0.5, delay=2, n_updates=2)
    gen = torch.Generator().manual_seed(1)
    actor = _rand_net([S, 256, 256, A], ["relu", "relu", "tanh"], gen)
    q1 = _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen)
    q2 = _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen)
    arrays = {}
    _net_arrays(arrays, "actor0", actor)
    _net_arrays(arrays, "q1_0", q1)
    _net_arrays(arrays, "q2_0", q2)
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             action=torch.rand(B, A, generator=gen) * 1.98 - 0.99,
             next_action=torch.zeros(B, A), reward=torch.randn(B, 1, generator=gen),
             not_terminal=(torch.rand(B, 1, generator=gen) > 0.005).float())
    t = _build_td3(meta, arrays)
    st = O.Td3State(actor, q1, q2, lr=1e-3)
    gb = _pbatch({k: v.cuda() for k, v in b.items()})
    for it in range(meta["n_updates"]):
        nn_ = torch.randn(B, A, generator=gen)
        arrays[f"noise{it}.next"] = nn_.numpy()
        _inject(t, arrays, it)
        out = O.td3_update(st, b, nn_, it, gamma=0.99, tau=0.005)
        if it == 0:
            t._critic_step(gb, t.actor_network_target, t.q1_network_target,
                           t.q2_network_target, t._fill)
            for pi, g in enumerate(t.net_grads(t.q1_network)):
                G.grad_close(g, out["grads"]["q1"][pi], ("q1 grad", pi))
        closs, aloss = t.train_batch(gb, it)
        assert abs(float(closs[0]) - out["losses"][0]) <= TOL * max(1.0, abs(out["losses"][0]))
        if it == 0:
            assert G.rel_err(t._ws["td_target"], out["target"].reshape(-1)) < TOL
    for net, onet in ((t.q1_network, st.q1), (t.actor_network, st.actor)):
        for i, seq in enumerate(net.fc.dnn):
            _adam_close(seq[0].weight, onet["W"][i], meta)
    for i, seq in enumerate(t.actor_network_target.fc.dnn):
        _adam_close(seq[0].weight, st.actor_t["W"][i], meta)
