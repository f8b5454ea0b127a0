"""The cross-entropy-method planner on the H100: rb200_cem_rollout against the reference's
goldens and the fp64 oracle, the zero-state equivalence with MemoryNetwork.forward, the shape
edges, reproducibility, no host synchronisation, and CEMTrainer / CrossEntropyMethod."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cem_oracle  # noqa: E402
from oracle import mdnrnn_oracle as mo  # noqa: E402
from tests.cem_cases import (CASES, TRAINER_CASES, assert_plans_match, noise_of,  # noqa: E402
                             planner_of, seeded_world_models)
from tests.golden_util import _adam_close, load  # noqa: E402

from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import (CEMTrainerParameters, MDNRNNTrainerParameters,  # noqa: E402
                                          NormalizationData, NormalizationKey,
                                          NormalizationParameters, RLParameters)
from reagent_b200.models import CEMPlannerNetwork, MemoryNetwork  # noqa: E402
from reagent_b200.models.cem_planner import PHI_LO, PHI_WIDTH  # noqa: E402

pytestmark = pytest.mark.gpu


def _plan_dict(planner, state, noise_arrays, dump=None):
    noise = planner.new_noise(state.device).copy_(**noise_arrays)
    p = planner.plan(state, noise=noise, dump=dump)
    n = int(p.n_iters.item())
    out = dict(values=p.values[:n].cpu().numpy(), n_iters=n)
    if planner.discrete_action:
        out.update(action=int(p.action.item()), one_hot=p.one_hot.cpu().numpy())
    else:
        out.update(elites=p.elites[:n].cpu().numpy(), mean=p.mean[:n].cpu().numpy(),
                   var=p.var[:n].cpu().numpy(), action=p.action.cpu().numpy())
    return out


@pytest.mark.parametrize("name", CASES)
def test_golden_plan(name):
    arrays, meta = load(name)
    nets = [n.cuda() for n in seeded_world_models(arrays, meta)]
    planner = planner_of(nets, meta)
    state = torch.from_numpy(arrays["state"]).cuda()[None]
    got = _plan_dict(planner, state, noise_of(arrays))
    assert got["n_iters"] == meta["n_iters"]
    assert_plans_match(got, arrays, meta["discrete"], name)
    if meta["discrete"]:
        np.testing.assert_array_equal(got["one_hot"], arrays["one_hot"])
    # forward returns the reference's types, on the CPU
    torch.manual_seed(0)
    out = planner(rlt.FeatureData(state))
    if meta["discrete"]:
        assert isinstance(out[0], int) and out[1].dtype == torch.float32 and out[1].device.type == "cpu"
    else:
        assert out.dtype == torch.float64 and tuple(out.shape) == (meta["A"],)


@pytest.mark.parametrize("name", CASES)
def test_zero_state_steps_equal_memory_network_forward(name):
    """Every step of iteration 0 is MemoryNetwork.forward on a [1, n, .] input from zeros: the
    rows of model m in the order the rollout groups them, bit for bit."""
    arrays, meta = load(name)
    nets = [n.cuda() for n in seeded_world_models(arrays, meta)]
    planner = planner_of(nets, meta)
    S, A, G, P, H = meta["S"], meta["A"], meta["G"], meta["P"], meta["H"]
    NG, DX = (2 * S + 1) * G + 2, S + A
    dump = torch.full((P, H, DX + NG), float("nan"), device="cuda")
    _plan_dict(planner, torch.from_numpy(arrays["state"]).cuda()[None], noise_of(arrays), dump)
    midx = torch.from_numpy(arrays["noise.model_idx"][0]).long()
    checked = 0
    for m, net in enumerate(nets):
        rows = torch.nonzero(midx == m).reshape(-1).cuda()
        for j in range(H):
            rec = dump[rows, j]
            ran = ~torch.isnan(rec[:, 0])
            if not bool(ran.any()):
                continue
            x = torch.nan_to_num(rec[:, :DX])
            out = net(rlt.FeatureData(x[None, :, A:].contiguous()),
                      rlt.FeatureData(x[None, :, :A].contiguous()))
            GS = G * S
            want = torch.cat([out.mus[0].reshape(-1, GS), out.sigmas[0].reshape(-1, GS),
                              out.logpi[0], out.reward[0, :, None], out.not_terminal[0, :, None]], 1)
            assert torch.equal(rec[ran, DX:], want[ran]), (name, m, j)
            checked += int(ran.sum())
    assert checked >= P


def _random_nets(K, S, A, Hd, L, G, seed, nt_bias=None):
    torch.manual_seed(seed)
    nets = []
    for _ in range(K):
        net = MemoryNetwork(S, A, Hd, L, G)
        with torch.no_grad():
            for p in net.mdnrnn.parameters():
                p.mul_(2.0)
            if nt_bias is not None:
                net.mdnrnn.gmm_linear.bias[-1] = nt_bias
        nets.append(net)
    P64 = [[p.detach().double().clone() for p in n.mdnrnn.parameters()] for n in nets]
    return [n.cuda() for n in nets], P64


# name: (discrete, P, K, S, A, hidden, layers, G, H, gamma, E, iters, terminal, nt_bias)
EDGES = {
    "p1_h30": (True, 1, 1, 4, 2, 16, 1, 1, 30, 1.0, 1, 1, True, 3.0),
    "p15_k3_g5": (False, 15, 3, 5, 2, 32, 2, 5, 4, 1.0, 3, 4, False, None),
    "p17_g32_l4_h128": (True, 17, 3, 3, 3, 128, 4, 32, 5, 0.0, 1, 1, True, 2.0),
    "p100_sa256_h1": (False, 100, 1, 200, 56, 32, 1, 1, 1, 1.0, 10, 3, False, None),
    "p1024_k3_h30": (True, 1024, 3, 4, 2, 64, 2, 5, 30, 1.0, 1, 1, True, 4.0),
    "p1024_cont": (False, 1024, 1, 4, 2, 64, 2, 2, 3, 0.0, 100, 3, True, 4.0),
    "end_on_step0": (True, 100, 1, 4, 2, 32, 2, 2, 10, 1.0, 1, 1, True, -6.0),
}


@pytest.mark.parametrize("name", list(EDGES))
def test_shape_edges_against_oracle(name):
    disc, P, K, S, A, Hd, L, G, H, gamma, E, iters, term, nt_bias = EDGES[name]
    nets, P64 = _random_nets(K, S, A, Hd, L, G, seed=len(name), nt_bias=nt_bias)
    lower, upper = [-1.0 - 0.5 * i for i in range(A)], [1.0 + 0.25 * i for i in range(A)]
    cfg = dict(discrete=disc, K=K, P=P, H=H, A=A, S=S, L=L, G=G, iters=iters, num_elites=E,
               gamma=gamma, alpha=0.25, epsilon=1e-6, terminal_effective=term,
               lower=None if disc else lower, upper=None if disc else upper)
    rng = np.random.RandomState(P + H)
    state = rng.standard_normal(S).astype(np.float32).astype(np.float64)
    noise, want = cem_oracle.guard_noise(P64, cfg, state, cem_oracle.make_noise(rng, cfg), rng)
    planner = CEMPlannerNetwork(
        mem_net_list=nets, cem_num_iterations=iters, cem_population_size=P,
        ensemble_population_size=1, num_elites=E, plan_horizon_length=H, state_dim=S,
        action_dim=A, discrete_action=disc, terminal_effective=term, gamma=gamma, epsilon=1e-6,
        action_upper_bounds=None if disc else np.array(upper),
        action_lower_bounds=None if disc else np.array(lower))
    got = _plan_dict(planner, torch.tensor(state, dtype=torch.float32).cuda()[None], noise)
    assert got["n_iters"] == want["n_iters"]
    assert_plans_match(got, want, disc, name)
    if name == "end_on_step0":
        # most trajectories stop after their first step: their value is the one-step plan's
        one = {k: (v[:, :, :1] if k == "step" else v[:, :1] if k == "action_idx" else v)
               for k, v in noise.items()}
        first = cem_oracle.plan(P64, dict(cfg, H=1), state, one)["values"]
        assert (want["values"] == first).mean() > 0.9


def test_reproducible_under_manual_seed_and_noise_moments():
    arrays, meta = load("cem_linear_dynamics_many")
    planner = planner_of([n.cuda() for n in seeded_world_models(arrays, meta)], meta)
    state = torch.from_numpy(arrays["state"]).cuda()[None]
    runs = []
    for _ in range(2):
        torch.manual_seed(123)
        p = planner.plan(state)
        runs.append([t.clone() for t in (p.action, p.values, p.mean, p.var, p.elites)])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    torch.manual_seed(124)
    assert not torch.equal(planner.plan(state).values, runs[0][1])
    # the default noise: truncated normals in [-2, 2] with their moments, uniform indices
    torch.manual_seed(0)
    big = CEMPlannerNetwork([MemoryNetwork(4, 8, 8, 1, 1).cuda() for _ in range(4)], 10, 1024,
                            1, 10, 30, 4, 8, False, False, 1.0,
                            action_upper_bounds=np.ones(8), action_lower_bounds=-np.ones(8))
    z = big.new_noise(torch.device("cuda")).fill_().truncnorm.double()
    assert float(z.min()) >= -2.0 and float(z.max()) <= 2.0
    assert abs(float(z.mean())) < 3e-3
    assert abs(float(z.var()) - 0.7737413) < 3e-3  # 1 - 4 phi(2) / (Phi(2) - Phi(-2))
    assert abs(PHI_LO - 0.0227501319) < 1e-9 and abs(PHI_WIDTH - 0.9544997361) < 1e-9
    disc = CEMPlannerNetwork([MemoryNetwork(4, 4, 8, 1, 1).cuda() for _ in range(3)], 1, 1024,
                             1, 10, 30, 4, 4, True, False, 1.0)
    nz = disc.new_noise(torch.device("cuda")).fill_()
    cnt = torch.bincount(nz.action_idx.reshape(-1).long(), minlength=4).double()
    assert cnt.numel() == 4 and float((cnt / cnt.mean() - 1).abs().max()) < 0.05
    cnt = torch.bincount(nz.model_idx.reshape(-1).long(), minlength=3).double()
    assert cnt.numel() == 3 and float((cnt / cnt.mean() - 1).abs().max()) < 0.2
    u = nz.step[..., 0].double()
    assert 0.0 <= float(u.min()) and float(u.max()) < 1.0 and abs(float(u.mean()) - 0.5) < 0.01


def test_plan_does_not_synchronise():
    arrays, meta = load("cem_linear_dynamics_single")
    planner = planner_of([n.cuda() for n in seeded_world_models(arrays, meta)], meta)
    state = torch.from_numpy(arrays["state"]).cuda()[None]
    planner.plan(state)  # workspace and noise allocated
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(2_000_000_000)  # a spin kernel of ~1 s ahead of the plan on this stream
    p = planner.plan(state)
    assert not stream.query(), "plan() waited for the GPU"
    torch.cuda.synchronize()
    assert int(p.n_iters.item()) >= 1 and bool(torch.isfinite(p.action).all())


def _train_batch(arrays, it):
    g = lambda k: torch.from_numpy(arrays[f"batch{it}.{k}"]).cuda()  # noqa: E731
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(g("state")), next_state=rlt.FeatureData(g("next_state")),
        action=rlt.FeatureData(g("action")), reward=g("reward"), not_terminal=g("not_terminal"),
        time_diff=None, step=None)


def _cem_trainer(arrays, meta):
    from reagent_b200.training import CEMTrainer, MDNRNNTrainer

    nets = [n.cuda() for n in seeded_world_models(arrays, meta)]
    mdn = MDNRNNTrainerParameters(hidden_size=meta["hidden"], num_hidden_layers=meta["layers"],
                                  num_gaussians=meta["G"], action_dim=meta["A"],
                                  not_terminal_loss_weight=meta["not_terminal_weight"])
    trainers = [MDNRNNTrainer(n, mdn) for n in nets]
    return CEMTrainer(planner_of(nets, meta), trainers, CEMTrainerParameters(mdnrnn=mdn))


def _weights_close(tr, arrays, meta, t):
    m_ = dict(meta, n_updates=t)
    for m, wt in enumerate(tr.world_model_trainers):
        for i, p in enumerate(wt.memory_network.mdnrnn.parameters()):
            _adam_close(mo.sample(p.detach()), torch.from_numpy(arrays[f"p{t}.{m}.{i}"]), m_)


@pytest.mark.parametrize("name", TRAINER_CASES)
@pytest.mark.parametrize("fast", [False, True])
def test_trainer_matches_golden(name, fast):
    arrays, meta = load(name)
    tr = _cem_trainer(arrays, meta)
    opts = tr.configure_optimizers()
    assert len(opts) == meta["K"]
    assert [o.arena for o in opts] == [t.memory_network.arena for t in tr.world_model_trainers]
    for it in range(meta["n_updates"]):
        batch = _train_batch(arrays, it)
        if fast:
            losses = [float(v[3]) for v in tr.train_batch(batch, it)]
        else:
            gen = tr.train_step_gen(batch, it)
            losses = []
            for opt in tr.optimizers():
                loss = next(gen)
                opt.zero_grad()
                loss.backward()
                opt.step()
                losses.append(float(loss.detach()))
            with pytest.raises(StopIteration):
                next(gen)
        want = arrays["losses"][it]
        assert np.abs(np.array(losses) - want).max() <= 1e-5 * max(1.0, np.abs(want).max())
        _weights_close(tr, arrays, meta, it + 1)


def _norm(S, A, discrete, lo=-3.0, hi=3.0):
    state = {i: NormalizationParameters(feature_type="CONTINUOUS") for i in range(S)}
    if discrete:
        action = {100 + i: NormalizationParameters(feature_type="DISCRETE_ACTION") for i in range(A)}
    else:
        action = {100 + i: NormalizationParameters(feature_type="CONTINUOUS_ACTION", min_value=lo,
                                                   max_value=hi) for i in range(A)}
    return {NormalizationKey.STATE: NormalizationData(dense_normalization_parameters=state),
            NormalizationKey.ACTION: NormalizationData(dense_normalization_parameters=action)}


# the reference's three CEM configurations (configs/world_model/cem_*.yaml)
CONFIGS = {
    "cem_cartpole_offline": (1, 200.0, True),
    "cem_linear_dynamics_single": (1, 0.0, False),
    "cem_linear_dynamics_many": (2, 0.0, False),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_manager_builds_reference_configurations(name):
    from reagent_b200.model_managers import CEMPolicy, CrossEntropyMethod
    from reagent_b200.training import CEMTrainer

    K, ntw, discrete = CONFIGS[name]
    arrays, meta = load(name)
    S, A = meta["S"], meta["A"]
    manager = CrossEntropyMethod(trainer_param=CEMTrainerParameters(
        plan_horizon_length=meta["H"], num_world_models=K, cem_population_size=100,
        cem_num_iterations=10, ensemble_population_size=1, num_elites=15,
        mdnrnn=MDNRNNTrainerParameters(hidden_size=100, num_hidden_layers=2, learning_rate=0.001,
                                       not_terminal_loss_weight=ntw, next_state_loss_weight=1.0,
                                       reward_loss_weight=1.0, num_gaussians=1),
        rl=RLParameters(gamma=1.0, softmax_policy=False)))
    torch.manual_seed(meta["seed"])
    tr = manager.build_trainer(_norm(S, A, discrete), use_gpu=True)
    assert isinstance(tr, CEMTrainer) and len(tr.world_model_trainers) == K
    for m, t in enumerate(tr.world_model_trainers):
        for i, p in enumerate(t.memory_network.mdnrnn.parameters()):
            np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{m}.{i}.sha256"])
    pl = tr.cem_planner_network
    assert (pl.discrete_action, pl.terminal_effective, pl.state_dim, pl.action_dim) == (
        discrete, ntw > 0, S, A)
    if not discrete:
        np.testing.assert_array_equal(pl.action_upper_bounds, np.full(A * meta["H"], 3.0))
    policy = manager.create_policy(tr)
    assert isinstance(policy, CEMPolicy)
    out = policy.act(rlt.FeatureData(torch.randn(1, S, device="cuda")))
    assert tuple(out.action.shape) == (1, A) and out.action.device.type == "cpu"
    assert float(out.log_prob) == 0.0
    if discrete:
        assert float(out.action.sum()) == 1.0
    else:
        assert out.action.dtype == torch.float64 and float(out.action.abs().max()) <= 1.0
