"""GPU parity of SACTrainer with a state-value network and CRR weighting: the generator path
and train_batch against golden vectors of the unmodified reference (oracle/
make_sac_value_golden.py), the SAC manager at the reference's Pendulum configurations, the
config-4 per-GPU shape against the oracle, prioritized replay, the captured online step and
the C ABI's rejections.  Tolerances as in tests/test_actor_critic_gpu.py."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from oracle import sac_value_oracle as V
from tests import golden_util as G
from tests.online_step import assert_captured_equals_eager, tree
from tests.builders import _net_arrays, _pbatch, _rand_net
from tests.golden_cases import SAC_VALUE_CASES, opt_names
from tests.golden_util import _adam_close, _cmp_module

pytestmark = pytest.mark.gpu
TOL = 1e-5
E_INVALID = -1  # RB200_E_INVALID, include/reagent_b200.h


def _crr(meta):
    from reagent_b200.training import CRRWeightFn

    return None if meta["crr"] is None else CRRWeightFn(**meta["crr"])


def _build(meta, arrays):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import SACTrainer

    S, A, sz, ac = meta["S"], meta["A"], meta["sizes"], meta["acts"]
    actor = GaussianFullyConnectedActor(S, A, sz, ac)
    q1 = FullyConnectedCritic(S, A, sz, ac)
    q2 = FullyConnectedCritic(S, A, sz, ac) if meta["twin"] else None
    value = FloatFeatureFullyConnected(S, 1, sz, ac)
    G.load_into_module(arrays, "actor0", actor)
    G.load_into_module(arrays, "q1_0", q1)
    if q2 is not None:
        G.load_into_module(arrays, "q2_0", q2)
    G.load_into_module(arrays, "v0", value)
    opt = lambda: Optimizer__Union.default(lr=meta["lr"])  # noqa: E731
    t = SACTrainer(actor, q1, q2, value,
                   rl=RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"]),
                   q_network_optimizer=opt(), value_network_optimizer=opt(),
                   actor_network_optimizer=opt(),
                   alpha_optimizer=opt() if meta["learn_alpha"] else None,
                   minibatch_size=meta["B"], entropy_temperature=meta["entropy_temperature"],
                   logged_action_uniform_prior=meta["uniform_prior"],
                   target_entropy=meta["target_entropy"], crr_config=_crr(meta))
    return t.cuda()


def _build_manager(meta, arrays):
    """model_managers.SAC from the fields of the reference's Pendulum YAMLs."""
    from reagent_b200.core.parameters import (NormalizationData, NormalizationKey,
                                              NormalizationParameters, RLParameters)
    from reagent_b200.model_managers import SAC
    from reagent_b200.net_builder import (GaussianFullyConnected, ParametricFullyConnected,
                                          ValueFullyConnected)
    from reagent_b200.optimizer import Optimizer__Union

    fc = dict(sizes=[64, 64], activations=["leaky_relu", "leaky_relu"])
    kw = dict(rl=RLParameters(gamma=0.99, target_update_rate=0.005, softmax_policy=True),
              entropy_temperature=0.3,
              q_network_optimizer=Optimizer__Union.default(lr=0.001),
              value_network_optimizer=Optimizer__Union.default(lr=0.001),
              actor_network_optimizer=Optimizer__Union.default(lr=0.001),
              actor_net_builder=GaussianFullyConnected(**fc),
              critic_net_builder=ParametricFullyConnected(**fc),
              value_net_builder=ValueFullyConnected(**fc), minibatch_size=256)
    if meta["crr"] is not None:
        kw["crr_config"] = _crr(meta)
    else:
        kw["alpha_optimizer"] = Optimizer__Union.default(lr=0.001)
    norm = lambda n: NormalizationData(dense_normalization_parameters={  # noqa: E731
        i: NormalizationParameters(feature_type="CONTINUOUS", mean=0.0, stddev=1.0)
        for i in range(n)})
    t = SAC(**kw).build_trainer({NormalizationKey.STATE: norm(meta["S"]),
                                 NormalizationKey.ACTION: norm(meta["A"])}, use_gpu=True)
    with torch.no_grad():
        for net, prefix in ((t.actor_network, "actor0"), (t.q1_network, "q1_0"),
                            (t.q2_network, "q2_0"), (t.value_network, "v0")):
            for i, seq in enumerate(net.fc.dnn):
                seq[0].weight.copy_(torch.from_numpy(arrays[f"{prefix}.W{i}"]))
                seq[0].bias.copy_(torch.from_numpy(arrays[f"{prefix}.b{i}"]))
        for p, q in zip(t.value_network_target.parameters(), t.value_network.parameters()):
            p.copy_(q)
    return t


def _inject(t, arrays, it):
    def hook(name, shape, device):
        assert name == "cur", "a value network draws no noise for s'"
        return torch.from_numpy(arrays[f"noise{it}.cur"]).to(device)
    t.noise_hook = hook


def _check_final(t, arrays, meta):
    _cmp_module(t.actor_network, arrays, "actorN", 2e-5)
    _cmp_module(t.q1_network, arrays, "q1_N")
    if meta["twin"]:
        _cmp_module(t.q2_network, arrays, "q2_N")
    _cmp_module(t.value_network, arrays, "vN")
    _cmp_module(t.value_network_target, arrays, "vt_N")
    if meta["learn_alpha"]:
        assert G.rel_err(t.log_alpha, arrays["log_alpha_N"]) < TOL


def _close(got, ref, tol):
    assert abs(float(got) - ref) <= tol * max(1.0, abs(ref)), (float(got), ref)


def _run_generator(t, arrays, meta):
    from reagent_b200.training import run_update

    batch = _pbatch(G.batch_tensors(arrays, "cuda"))
    names = opt_names(meta)
    nets = {"q1": t.q1_network, "q2": t.q2_network, "actor": t.actor_network,
            "value": t.value_network}
    for it in range(meta["n_updates"]):
        _inject(t, arrays, it)
        if it == 0:
            opts = t.optimizers()
            assert len(opts) == len(names) + 1
            for oi, opt in enumerate(opts):
                loss = t.training_step(batch, it, oi)
                if oi < len(names):
                    nm = names[oi]
                    if nm == "alpha":
                        assert G.rel_err(t._ws["alpha_grad"], arrays[f"grad0.opt{oi}.0"]) < TOL
                    else:
                        tol = 5e-5 if nm == "actor" else TOL
                        for pi, g in enumerate(t.net_grads(nets[nm])):
                            assert G.rel_err(g, arrays[f"grad0.opt{oi}.{pi}"]) < tol, (nm, pi)
                    _close(loss.detach(), arrays["losses"][it][oi], TOL)
                opt.zero_grad()
                loss.backward()
                opt.step()
        else:
            losses = run_update(t, batch, it)
            for oi, ref in enumerate(arrays["losses"][it]):
                _close(losses[oi].detach(), ref, 2e-5)
    _check_final(t, arrays, meta)


def _run_fast(t, arrays, meta):
    batch = _pbatch(G.batch_tensors(arrays, "cuda"))
    names = opt_names(meta)
    for it in range(meta["n_updates"]):
        _inject(t, arrays, it)
        closs, aloss = t.train_batch(batch, it)
        ref = arrays["losses"][it]
        _close(closs[0], ref[0], 2e-5)
        _close(aloss[0], ref[names.index("actor")], 2e-5)
        _close(t._ws["value_loss"][0], ref[names.index("value")], 2e-5)
    _check_final(t, arrays, meta)


@pytest.mark.parametrize("name", SAC_VALUE_CASES)
def test_generator_path_matches_reference(name):
    arrays, meta = G.load(name)
    _run_generator(_build(meta, arrays), arrays, meta)


@pytest.mark.parametrize("name", SAC_VALUE_CASES)
def test_fast_path_matches_reference(name):
    arrays, meta = G.load(name)
    _run_fast(_build(meta, arrays), arrays, meta)


@pytest.mark.parametrize("name", ["sac_pendulum_manager", "sac_crr_pendulum_manager"])
@pytest.mark.parametrize("fast", [False, True])
def test_manager_pendulum_configs_match_reference(name, fast):
    arrays, meta = G.load(name)
    t = _build_manager(meta, arrays)
    assert sorted(t.state_dict().keys()) == meta["state_dict_keys"]
    (_run_fast if fast else _run_generator)(t, arrays, meta)


def _config4(crr, uniform_prior=True, weighted=False):
    """BASELINE config 4 per-GPU shard: S=256, A=32, B=2048, [256,256] networks."""
    S, A, B = 256, 32, 2048
    crr_kw = dict(exponent_beta=1.0, exponent_clamp=20.0) if crr else None
    meta = dict(S=S, A=A, B=B, sizes=[256, 256], acts=["relu", "relu"], twin=True,
                learn_alpha=True, gamma=0.99, tau=0.005, lr=1e-3, entropy_temperature=0.1,
                target_entropy=-float(A), uniform_prior=uniform_prior, crr=crr_kw, n_updates=2)
    gen = torch.Generator().manual_seed(2)
    nets = dict(actor0=_rand_net([S, 256, 256, 2 * A], ["relu", "relu", "linear"], gen),
                q1_0=_rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen),
                q2_0=_rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen),
                v0=_rand_net([S, 256, 256, 1], ["relu", "relu", "linear"], gen))
    arrays = {}
    for k, n in nets.items():
        _net_arrays(arrays, k, n)
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             action=torch.rand(B, A, generator=gen) * 1.98 - 0.99,
             next_action=torch.zeros(B, A), reward=torch.randn(B, 1, generator=gen),
             not_terminal=(torch.rand(B, 1, generator=gen) > 0.005).float())
    w = (torch.rand(B, generator=gen) + 0.25) if weighted else None
    t = _build(meta, arrays)
    st = V.SacValueState(nets["actor0"], nets["q1_0"], nets["q2_0"], nets["v0"], lr=1e-3,
                         entropy_temperature=0.1, learn_alpha=True, target_entropy=-float(A),
                         logged_action_uniform_prior=uniform_prior, crr=crr_kw)
    gb = _pbatch({k: v.cuda() for k, v in b.items()})
    for it in range(meta["n_updates"]):
        nc = torch.randn(B, A, generator=gen)
        arrays[f"noise{it}.cur"] = nc.numpy()
        _inject(t, arrays, it)
        out = V.sac_value_update(st, b, nc, gamma=0.99, tau=0.005, sample_weight=w)
        if it == 0:
            t._critic_step(gb, t.actor_network, None, None, t._fill_critic)
            for pi, g in enumerate(t.net_grads(t.q1_network)):
                if not weighted:
                    G.grad_close(g, out["grads"]["q1"][pi], ("q1 grad", pi))
            assert G.rel_err(t._ws["td_target"], out["target"].reshape(-1)) < TOL
        closs, aloss = t.train_batch(gb, it, importance_weights=None if w is None else w.cuda())
        # from update 1 on both sides start from post-Adam weights that agree only within the
        # _adam_close budget (an element with a gradient at fp32 noise can move by lr either way)
        tol = 2e-5 if it == 0 else 1e-4
        for got, ref in ((closs[0], out["losses"][0]), (closs[1], out["losses"][1]),
                         (aloss[0], out["losses"][2]), (t._ws["value_loss"][0], out["losses"][4])):
            _close(got, ref, tol)
        if weighted and it == 0:
            assert G.rel_err(t._ws["td_error"], out["td_error"].cuda()) < 5e-5
    for net, onet in ((t.q1_network, st.q1), (t.actor_network, st.actor),
                      (t.value_network, st.value), (t.value_network_target, st.value_t)):
        for i, seq in enumerate(net.fc.dnn):
            _adam_close(seq[0].weight, onet["W"][i], meta)
    assert G.rel_err(t.log_alpha, st.log_alpha) < TOL


@pytest.mark.parametrize("crr", [False, True])
def test_config4_shard_matches_oracle(crr):
    _config4(crr)


def test_config4_learnable_alpha_entropy_value_target_matches_oracle():
    """logged_action_uniform_prior=False with a learnable alpha: the value target uses the
    post-update alpha (the reference cannot backpropagate this case: its target is float64)."""
    _config4(False, uniform_prior=False)


def test_config4_importance_weights_match_weighted_oracle():
    _config4(False, weighted=True)


def test_no_value_network_keeps_q_targets():
    arrays, meta = G.load("sac_value_twin_alpha")
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.training import SACTrainer

    S, A, sz, ac = meta["S"], meta["A"], meta["sizes"], meta["acts"]
    t = SACTrainer(GaussianFullyConnectedActor(S, A, sz, ac), FullyConnectedCritic(S, A, sz, ac),
                   FullyConnectedCritic(S, A, sz, ac)).cuda()
    keys = t.state_dict().keys()
    assert any(k.startswith("q1_network_target") for k in keys)
    assert not any(k.startswith("value_network") for k in keys)


# ---------------------------------------------------------------------------
# the captured online step
# ---------------------------------------------------------------------------
def _online_setup(base, cfg, crr):
    from reagent_b200.replay_memory import PrioritizedReplayBuffer

    S, A = cfg["S"], cfg["A"]
    meta = dict(S=S, A=A, B=cfg["B"], sizes=[256, 256], acts=["relu", "relu"], twin=True,
                learn_alpha=True, gamma=0.99, tau=0.005, lr=1e-3, entropy_temperature=0.1,
                target_entropy=-float(A), uniform_prior=True,
                crr=dict(exponent_beta=1.0, exponent_clamp=20.0) if crr else None)
    gen = torch.Generator().manual_seed(4)
    arrays = {}
    _net_arrays(arrays, "actor0", _rand_net([S, 256, 256, 2 * A], ["relu", "relu", "linear"], gen))
    _net_arrays(arrays, "q1_0", _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen))
    _net_arrays(arrays, "q2_0", _rand_net([S + A, 256, 256, 1], ["relu", "relu", "linear"], gen))
    _net_arrays(arrays, "v0", _rand_net([S, 256, 256, 1], ["relu", "relu", "linear"], gen))
    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=cfg["cap"], batch_size=cfg["B"])
    rb.add_batch(**base)
    return rb, _build(meta, arrays)


def _state(t):
    out = [p.detach().clone() for p in t.parameters()]
    return out + [b.detach().clone() for b in t.buffers()]


@pytest.mark.parametrize("with_per", [False, True])
@pytest.mark.parametrize("crr", [False, True])
def test_online_captured_equals_eager(crr, with_per):
    """FusedPolicyStep with a value network: graph replay and eager launches of the same update
    from identical states and noise agree bit for bit (losses, every network, the tree)."""
    import bench
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedPolicyStep

    cfg = dict(bench.CONFIGS[4], cap=4096, B=256)
    low, high = -np.ones(cfg["A"], np.float32), np.ones(cfg["A"], np.float32)
    base = bench.synth_stream(3000, 7, cfg)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=10, eps=1e-6) if with_per else None
    draws = []  # the noise each run asked its hook for

    def setup():
        rb, t = _online_setup(base, cfg, crr)
        gen = torch.Generator().manual_seed(11)
        buf = torch.empty(cfg["B"], cfg["A"], device="cuda")
        draws.append([])

        def hook(name, shape, device):
            draws[-1].append(name)
            return buf
        t.noise_hook = hook

        def refill():
            torch.cuda.synchronize()
            buf.copy_(torch.randn(buf.shape, generator=gen))
        refill()
        random.seed(5)
        return FusedPolicyStep(t, rb, cfg["B"], low, high, online=True, per=per), refill

    snap = assert_captured_equals_eager(
        setup, bench.synth_stream(5, 8, cfg), 5,
        lambda f: [_state(f.trainer), tree(f), f.trainer.all_batches_processed],
        scalar_loss=False)
    assert [set(d) for d in draws] == [{"cur"}, {"cur"}]
    assert snap[-1] == 6


def test_online_per_write_back_is_twin_critic_priority():
    import bench
    from oracle import per_ac_oracle as PA
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedPolicyStep

    cfg = dict(bench.CONFIGS[4], cap=4096, B=256)
    low, high = -np.ones(cfg["A"], np.float32), np.ones(cfg["A"], np.float32)
    rb, t = _online_setup(bench.synth_stream(3000, 3, cfg), cfg, crr=True)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=20, eps=1e-6)
    random.seed(77)
    fused = FusedPolicyStep(t, rb, cfg["B"], low, high, online=True, per=per)
    extra = bench.synth_stream(3, 4, cfg)
    for i in range(3):
        fused.step({k: v[i] for k, v in extra.items()})
        torch.cuda.synchronize()
        ws = t._ws
        want = PA.twin_td_priorities(ws["q1_value"].cpu().numpy(), ws["q2_value"].cpu().numpy(),
                                     ws["td_target"].cpu().numpy(), per.alpha, per.eps)
        got = fused.priorities.cpu().numpy()
        assert np.allclose(got, want, rtol=1e-6, atol=0)


# ---------------------------------------------------------------------------
# C ABI rejections
# ---------------------------------------------------------------------------
def _abi_setup():
    arrays, meta = G.load("sac_crr_exponent")
    t = _build(meta, arrays)
    batch = _pbatch(G.batch_tensors(arrays, "cuda"))
    _inject(t, arrays, 0)
    t.train_batch(batch, 0)  # workspaces
    return t, batch, meta


def _args(t, batch):
    from reagent_b200.training.workspace import Pins

    pins = Pins(batch.state.float_features.device)
    a, _ = t._base_args(batch, t._ws, pins)
    a.loss = t._ws["critic_loss"].data_ptr()
    t._fill_actor(a, pins)
    a.noise_next = a.noise_cur
    return a, pins


def test_c_abi_rejects_bad_value_networks():
    from reagent_b200 import _lib
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected

    t, batch, meta = _abi_setup()
    lib, st = _lib.lib(), _lib.cur_stream()
    S = meta["S"]
    d = lambda n: n.arena.desc()  # noqa: E731
    ws = t._ws
    wide = FloatFeatureFullyConnected(S + 1, 1, [8], ["relu"]).cuda()
    two = FloatFeatureFullyConnected(S, 2, [8], ["relu"]).cuda()

    def critic(a):
        return lib.rb200_ac_critic_step(d(t.actor_network), d(t.q1_network), d(t.q2_network),
                                        None, None, a, ws["q1"].c, ws["q2"].c, st)

    def actor(a):
        return lib.rb200_ac_actor_step(d(t.actor_network), d(t.q1_network), d(t.q2_network), a,
                                       ws["actor"].c, ws["q1"].c, ws["q2"].c, st)

    # critic step: the value target's widths, and a value network with TD3
    for net in (wide, two):
        a, pins = _args(t, batch)
        a.value_target = C.pointer(d(net))
        assert critic(a) == E_INVALID
    a, pins = _args(t, batch)
    a.value_target = C.pointer(d(t.value_network_target))
    assert critic(a) == 0
    a.algo = _lib.ALGO_TD3
    assert critic(a) == E_INVALID
    # actor step: CRR without a value network, bad widths, without backprop through log_prob
    a, pins = _args(t, batch)
    a.value_net = None
    assert actor(a) == E_INVALID and b"value network" in lib.rb200_last_error()
    for net in (wide, two):
        a, pins = _args(t, batch)
        a.value_net = C.pointer(d(net))
        assert actor(a) == E_INVALID
    a, pins = _args(t, batch)
    a.backprop_through_log_prob = 0
    assert actor(a) == E_INVALID
    a, pins = _args(t, batch)
    assert actor(a) == 0
    # value step: a null descriptor, bad widths, TD3, a missing min_q
    a, pins = _args(t, batch)
    a.loss = ws["value_loss"].data_ptr()
    a.logged_action_uniform_prior = 0  # the entropy target needs log_prob_out
    assert lib.rb200_ac_value_step(d(t.value_network), a, ws["value"].c, st) == E_INVALID
    a.logged_action_uniform_prior = 1
    assert lib.rb200_ac_value_step(None, a, ws["value"].c, st) == E_INVALID
    assert lib.rb200_ac_value_step(d(two), a, ws["value"].c, st) == E_INVALID
    assert lib.rb200_ac_value_step(d(t.value_network), a, ws["value"].c, st) == 0
    a.algo = _lib.ALGO_TD3
    assert lib.rb200_ac_value_step(d(t.value_network), a, ws["value"].c, st) == E_INVALID
    a.algo = _lib.ALGO_SAC
    a.min_q_out = None
    assert lib.rb200_ac_value_step(d(t.value_network), a, ws["value"].c, st) == E_INVALID
    torch.cuda.synchronize()
