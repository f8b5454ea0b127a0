"""REINFORCE and PPO without a GPU: the plain-torch restatement (oracle/pg_oracle.py) against
every golden of the unmodified reference, regeneration from the reference, constructor and
manager defaults, the yield counts and optimizer order, and the refusals."""
import glob
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import pg_oracle as PO
from oracle import td_oracle as O
from oracle.ref_harness import reference_available
from tests import golden_util as G
from tests import pg_cases as P


@pytest.mark.parametrize("name", P.REINFORCE_CASES)
def test_reinforce_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    pol, val = P.oracle_nets(arrays, meta)
    ap, av = P.adam(meta, pol), P.adam(meta, val)
    for u, t in enumerate(P.trajectories(arrays)):
        losses, grads, ret, _ = PO.reinforce_update(pol, val, ap, av, t, **P.reinforce_kwargs(meta))
        assert torch.equal(ret, torch.from_numpy(arrays[f"dret{u}"])), "returns are bit-identical"
        P.check_losses(losses, arrays["losses"][u])
        if u == 0:
            for oi, g in enumerate(grads):
                P.check_grads(arrays, oi, g)
        P.check_net(arrays, f"policy{u + 1}", O.net_params(pol))
        if val is not None:
            P.check_net(arrays, f"value{u + 1}", O.net_params(val))


@pytest.mark.parametrize("name", P.PPO_CASES)
def test_ppo_oracle_matches_reference(name):
    arrays, meta = G.load(name)
    pol, val = P.oracle_nets(arrays, meta)
    ap, av = P.adam(meta, pol), P.adam(meta, val)
    trajs = P.trajectories(arrays)
    n_adv = 0
    for m, (u, idx) in enumerate(P.minibatches(arrays, meta)):
        losses, grads, adv = PO.ppo_update(pol, val, ap, av, [trajs[i] for i in idx],
                                           **P.ppo_kwargs(meta))
        want = np.concatenate([arrays[f"adv{n_adv + j}"] for j in range(len(idx))])
        n_adv += len(idx)
        assert G.rel_err(adv, want) < G.TOL
        P.check_losses(losses, arrays["losses"][m])
        if m == 0:
            for oi, g in enumerate(grads):
                P.check_grads(arrays, oi, g)
        last = m + 1 == len(P.minibatches(arrays, meta)) or P.minibatches(arrays, meta)[m + 1][0] != u
        if last:
            P.check_net(arrays, f"policy{u + 1}", O.net_params(pol))
            if val is not None:
                P.check_net(arrays, f"value{u + 1}", O.net_params(val))


@pytest.mark.parametrize("name", P.PG_CASES)
def test_returns_fp64_matches_reference_returns(name):
    """The fp64 kernel reference against the reference's fp32 discounted_returns (PPO's TD
    advantage never calls it)."""
    arrays, meta = G.load(name)
    trajs = P.trajectories(arrays)
    if meta["kind"] == "ppo":
        order = [i for _, idx in P.minibatches(arrays, meta) for i in idx]
    else:
        order = list(range(len(trajs)))
    if meta["kind"] == "ppo" and meta["td_error_advantage"]:
        assert "dret0" not in arrays
        return
    for k, i in enumerate(order):
        r = trajs[i]["reward"]
        want = PO.discounted_returns(torch.clamp(r, max=meta["reward_clip"]), meta["gamma"])
        assert torch.equal(want, torch.from_numpy(arrays[f"dret{k}"]))
        got = PO.returns_fp64(r, [0, len(r)], gamma=meta["gamma"], reward_clip=meta["reward_clip"],
                              normalize=False, subtract_mean=False, offset_clamp_min=False)
        assert G.rel_err(got, want) < 1e-6


def test_whiten_length_one_and_constant_give_zero():
    for x in (torch.tensor([3.5]), torch.ones(6)):
        assert torch.equal(PO.whiten(x, True), torch.zeros_like(x))
        got = PO.returns_fp64(x, [0, len(x)], gamma=0.0, reward_clip=1e6, normalize=True,
                              subtract_mean=True, offset_clamp_min=False)
        assert torch.equal(got, torch.zeros(len(x), dtype=torch.float64))


def test_goldens_cover_the_cases():
    a, meta = G.load("pg_ppo_baseline_entropy_dueling")
    assert meta["dueling"] and meta["update_epochs"] == 2 and meta["update_freq"] == 5
    assert [len(x) for x in [a["perm0.0"], a["perm0.1"]]] == [5, 5]
    assert len(P.minibatches(a, meta)) == 4  # 3 + 2 per epoch: a short last minibatch
    # ratios on both sides of [0.8, 1.2] at the initial policy
    pol, _ = P.oracle_nets(a, meta)
    rhos = []
    for t in P.trajectories(a):
        lp = PO.log_prob(O.mlp(pol, t["state"]), t.get("possible_actions_mask"), t["action"],
                         meta["temperature"])
        rhos.append(torch.exp(lp - t["log_prob"]).detach())
    rho = torch.cat(rhos)
    assert bool((rho < 0.8).any()) and bool((rho > 1.2).any())
    a, meta = G.load("pg_ppo_td_next_state")
    assert {float(a[f"traj{k}.not_terminal"][-1]) for k in range(4)} == {0.0, 1.0}
    a, meta = G.load("pg_reinforce_whiten_offpolicy")
    assert a["traj1.state"].shape[0] == 1
    assert float(np.max(a["traj0.reward"])) > meta["reward_clip"]
    assert (a["traj0.possible_actions_mask"] == 0).any()


@pytest.mark.skipif(not reference_available(), reason="needs the reference checkout")
def test_goldens_regenerate_from_reference(tmp_path, monkeypatch):
    from oracle import make_golden, make_pg_golden

    monkeypatch.setattr(make_golden, "GOLDEN", str(tmp_path))
    make_pg_golden.main()
    for path in sorted(glob.glob(os.path.join(G.GOLDEN, "pg_*.npz"))):
        new = np.load(os.path.join(tmp_path, os.path.basename(path)))
        old = np.load(path)
        assert sorted(new.files) == sorted(old.files), path
        for k in old.files:
            assert np.array_equal(old[k], new[k], equal_nan=True), (path, k)


# ---------------------------------------------------------------------------
def _policy(S=5, A=3, dueling=False, temperature=1.0):
    from reagent_b200.gym.policies import Policy, SoftmaxActionSampler
    from reagent_b200.models import DuelingQNetwork, FullyConnectedDQN

    net = (DuelingQNetwork.make_fully_connected(S, A, [8, 8], ["relu", "relu"]) if dueling
           else FullyConnectedDQN(S, A, [8], ["relu"]))
    return Policy(scorer=net, sampler=SoftmaxActionSampler(temperature))


def _value(S=5):
    from reagent_b200.net_builder import ValueFullyConnected
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters

    nd = NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS") for i in range(S)})
    return ValueFullyConnected(sizes=[8], activations=["relu"]).build_value_network(nd)


@pytest.mark.skipif(not reference_available(), reason="needs the reference checkout")
@pytest.mark.parametrize("which", ["reinforce_trainer.ReinforceTrainer", "ppo_trainer.PPOTrainer"])
def test_constructor_defaults_match_reference(which):
    from oracle.ref_harness import ref
    from reagent_b200 import training

    mod, cls = which.split(".")
    theirs = inspect.signature(getattr(ref("reagent.training." + mod), cls).__init__).parameters
    ours = inspect.signature(getattr(training, cls).__init__).parameters
    assert list(ours) == list(theirs)
    for k, p in theirs.items():
        if isinstance(p.default, (bool, int, float)) or p.default is None:
            assert ours[k].default == p.default, k


def test_yields_and_optimizer_order():
    from reagent_b200.training import PPOTrainer, ReinforceTrainer

    t = ReinforceTrainer(_policy())
    assert len(t.configure_optimizers()) == 1
    t = ReinforceTrainer(_policy(), value_net=_value(), normalize=False, subtract_mean=False)
    opts = [o["optimizer"] for o in t.configure_optimizers()]
    assert [o.arena for o in opts] == [t.value_net.arena, t.scorer.arena]
    t = PPOTrainer(_policy(), value_net=_value(), normalize=False)
    opts = [o["optimizer"] for o in t.configure_optimizers()]
    assert [o.arena for o in opts] == [t.value_net.arena, t.scorer.arena]
    assert t.get_optimizers()[1] is t.optimizers()[1]
    assert PPOTrainer(_policy()).get_optimizers()[0] is None


def test_refusals():
    from reagent_b200.gym.policies import GreedyActionSampler, Policy
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import PPOTrainer, ReinforceTrainer
    from reagent_b200.training.policy_gradient import PackedTrajectories
    from reagent_b200.training.workspace import Pins
    from reagent_b200.core import types as rlt

    for cls in (ReinforceTrainer, PPOTrainer):
        with pytest.raises(NotImplementedError):
            cls(Policy(scorer=FullyConnectedDQN(5, 3, [8], ["relu"]), sampler=GreedyActionSampler()))
        with pytest.raises(NotImplementedError):
            cls(Policy(scorer=torch.nn.Linear(5, 3), sampler=_policy().sampler))
        with pytest.raises(NotImplementedError):
            cls(Policy(scorer=FullyConnectedDQN(5, 3, [8], ["relu"], num_atoms=4),
                       sampler=_policy().sampler))
    with pytest.raises(NotImplementedError):
        ReinforceTrainer(_policy(), do_log_metrics=True)
    with pytest.raises(RuntimeError):
        ReinforceTrainer(_policy(), value_net=_value())
    with pytest.raises(RuntimeError):
        ReinforceTrainer(_policy(), value_net=_value(), normalize=False)
    with pytest.raises(AssertionError):
        PPOTrainer(_policy(), value_net=_value())
    with pytest.raises(AssertionError):
        PPOTrainer(_policy(), td_error_advantage=True)
    # every packed field is checked against T, S = 5 and A = 3 before anything is launched
    def traj(T=4, S=5, A=3, **kw):
        d = dict(state=rlt.FeatureData(torch.zeros(T, S)), action=torch.zeros(T, A),
                 reward=torch.zeros(T), log_prob=torch.zeros(T))
        d.update(kw)
        return rlt.PolicyGradientInput(**d)

    def refused(t, match, log_prob=True, td=True):
        with pytest.raises(ValueError, match=match):
            PackedTrajectories([traj(), t], Pins(torch.device("cpu")), 5, 3, log_prob=log_prob,
                               td=td)

    refused(traj(T=0), "at least one step")
    refused(traj(action=torch.zeros(4)), "action has shape")
    refused(traj(action=torch.zeros(4, 2)), "action has shape")
    refused(traj(state=rlt.FeatureData(torch.zeros(6, 5))), "state has shape")
    refused(traj(state=rlt.FeatureData(torch.zeros(4, 6))), "state has shape")
    refused(traj(reward=torch.zeros(3)), "reward has shape")
    refused(traj(reward=torch.zeros(4, 1)), "reward has shape")
    refused(traj(log_prob=torch.zeros(5)), "log_prob has shape")
    refused(traj(possible_actions_mask=torch.ones(4, 2)), "possible_actions_mask has shape")
    refused(traj(next_state=rlt.FeatureData(torch.zeros(3, 5))), "next_state has shape")
    refused(traj(not_terminal=torch.ones(4, 1)), "not_terminal has shape")
    refused(traj(next_state=rlt.FeatureData(torch.zeros(4, 5))), "every trajectory")


def test_manager_defaults_and_cartpole_configs():
    from reagent_b200 import model_managers as M
    from reagent_b200.net_builder import Dueling, FullyConnected
    from reagent_b200.optimizer import Optimizer__Union

    for cls in (M.Reinforce, M.PPO):
        m = cls(actions=["0", "1"])
        assert isinstance(m.policy_net_builder, Dueling)
        assert m.value_net_builder is None and m.sampler_temperature == 1.0
        with pytest.raises(AssertionError, match="at least 2 actions"):
            cls(actions=["0"])
    assert M.Reinforce(actions=["0", "1"]).gamma == 0.0 and M.PPO(actions=["0", "1"]).gamma == 0.9
    # the CartPole configurations (S 4, A 2), built on the CPU without their trainers
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters

    nd = NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS") for i in range(4)})
    r = M.Reinforce(actions=["0", "1"], gamma=0.99, off_policy=False,
                    optimizer=Optimizer__Union.default(lr=0.001), normalize=False,
                    subtract_mean=True,
                    policy_net_builder=FullyConnected(sizes=[64], activations=["leaky_relu"]))
    p = M.PPO(actions=["0", "1"], gamma=0.99, ppo_epsilon=0.2,
              optimizer=Optimizer__Union.default(lr=0.001, weight_decay=0.001), update_freq=2,
              update_epochs=1, ppo_batch_size=2,
              policy_net_builder=FullyConnected(sizes=[32, 32],
                                                activations=["leaky_relu", "leaky_relu"]))
    for m, dims in ((r, [4, 64, 2]), (p, [4, 32, 32, 2])):
        net = m.policy_net_builder.build_q_network(None, nd, len(m.actions))
        assert net.arena.dims == dims
        pol = m._create_policy(net)
        assert m._create_policy(net) is pol and pol.scorer is net
        assert pol.sampler.temperature == 1.0
    with pytest.raises(RuntimeError, match="CUDA only"):
        r.build_trainer({"state": nd}, use_gpu=False)


def test_policy_gradient_input_from_dict():
    from reagent_b200.core import types as rlt

    d = dict(observation=torch.randn(4, 3), action=torch.eye(2)[[0, 1, 1, 0]],
             reward=torch.randn(4), log_prob=torch.randn(4), next_observation=torch.randn(4, 3))
    b = rlt.PolicyGradientInput.from_dict(d)
    assert len(b) == 4 and b.next_state is not None and b.not_terminal is None
    p = rlt.PolicyGradientInput.input_prototype()
    assert p.action.shape == (10, 2) and p.possible_actions_mask.shape == (10, 2)
