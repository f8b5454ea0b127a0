"""DiscreteCRRTrainer on the GPU against the goldens of the unmodified reference: the generator
under the Lightning-style loop and `train_batch`, bit equality of the two, the CartPole
configuration through the model manager, and FusedDqnStep against the loop it captures."""
import random

import numpy as np
import pytest
import torch

from tests import golden_util as G
from tests.online_step import assert_captured_equals_eager, params
from tests.golden_cases import (CRR_CASES, check_grads, check_losses, check_params, initial_tensors,
                                net_names, noise_of)

pytestmark = pytest.mark.gpu


def tols(meta):
    """(losses / gradients / weights, parameters).  1e-5 on the small cases.  The [1024, 1024]
    CartPole case contracts over 1024 3xTF32 products (~22 mantissa bits each): on an H100 its
    losses differ from the fp32 reference by up to 2.4e-5, its gradients by 2.1e-5 and its actor
    weights (an exponential of the advantage) by 4.5e-5.  Adam then divides every gradient entry
    by its own magnitude, so an entry within that error of zero takes a step of another size:
    after three updates one of the 31 k sampled parameters is off by 5.1e-4 of the tensor's
    largest, the others by less than 1e-4."""
    return (1e-4, 1e-3) if meta["compact"] else (1e-5, 1e-5)


def _optimizer(meta):
    from reagent_b200.optimizer import Optimizer__Union

    if meta["optimizer"] == "AdamW":
        return Optimizer__Union(AdamW=dict(lr=meta["lr"], **meta["opt_kw"]))
    return Optimizer__Union.default(lr=meta["lr"])


def _rl(meta):
    from reagent_b200.core.parameters import RLParameters

    return RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                        reward_boost=meta["boost"], temperature=meta["temperature"])


def _load(arrays, meta, name, module):
    with torch.no_grad():
        for p, v in zip(module.parameters(), initial_tensors(arrays, meta, name)):
            p.copy_(v.to(p.device))


def _networks(trainer):
    t = trainer
    return {"actor": t.actor_network, "actor_t": t.actor_network_target, "q1": t.q1_network,
            "q1_t": t.q1_network_target, "q2": t.q2_network, "q2_t": t.q2_network_target,
            "r": t.reward_network, "c": t.q_network_cpe, "ct": t.q_network_cpe_target}


def build_trainer(arrays, meta):
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import DuelingQNetwork, FullyConnectedActor, FullyConnectedDQN
    from reagent_b200.training import DiscreteCRRTrainer

    S, A, sizes, acts = meta["S"], meta["A"], meta["sizes"], meta["acts"]

    def critic():
        if meta["dueling"]:
            return DuelingQNetwork.make_fully_connected(S, A, sizes, acts).cuda()
        return FullyConnectedDQN(S, A, sizes, acts).cuda()

    actor = FullyConnectedActor(S, A, sizes, acts,
                                exploration_variance=meta["exploration_variance"]).cuda()
    q1 = critic()
    q2 = critic() if meta["twin"] else None
    cpe = meta["cpe_metrics"] is not None
    r = c = None
    if cpe:
        n_out = (len(meta["cpe_metrics"]) + 1) * A
        r = FullyConnectedDQN(S, n_out, sizes, acts).cuda()
        c = FullyConnectedDQN(S, n_out, sizes, acts).cuda()
    t = DiscreteCRRTrainer(
        actor_network=actor, actor_network_target=actor.get_target_network(), q1_network=q1,
        q1_network_target=q1.get_target_network(), reward_network=r, q2_network=q2,
        q2_network_target=None if q2 is None else q2.get_target_network(), q_network_cpe=c,
        q_network_cpe_target=None if c is None else c.get_target_network(),
        metrics_to_score=meta["cpe_metrics"],
        evaluation=EvaluationParameters(calc_cpe_in_training=cpe), rl=_rl(meta),
        double_q_learning=meta["twin"], q_network_optimizer=_optimizer(meta),
        actor_network_optimizer=_optimizer(meta), use_target_actor=meta["use_target_actor"],
        actions=[str(i) for i in range(A)], delayed_policy_update=meta["delayed_policy_update"],
        beta=meta["beta"], entropy_coeff=meta["entropy_coeff"], clip_limit=meta["clip_limit"],
        max_weight=meta["max_weight"]).cuda()
    for name, net in _networks(t).items():
        if net is not None:
            _load(arrays, meta, name, net)
    return t


def rlt_batch(arrays, device="cuda"):
    from reagent_b200.core import types as rlt

    b = G.batch_tensors(arrays, device)
    return rlt.DiscreteDqnInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
        reward=b["reward"], time_diff=torch.ones_like(b["reward"]), step=None,
        not_terminal=b["not_terminal"], action=b["action"],
        next_action=torch.zeros_like(b["action"]),
        possible_actions_mask=torch.ones_like(b["action"]),
        possible_next_actions_mask=b["possible_next_actions_mask"],
        extras=rlt.ExtraData(action_probability=b["action_probability"],
                             metrics=b.get("metrics")))


def inject_noise(trainer, arrays, meta, it):
    """The reference's draws of update `it`, as the N(0, 1) draw the trainer then scales."""
    scale = meta["exploration_variance"]
    if scale is None:
        return
    draws = {"next": noise_of(arrays, it, "next", "cuda"), "cur": noise_of(arrays, it, "cur", "cuda")}
    trainer.noise_hook = lambda name, shape, device: draws[name] / scale


def _final_check(t, arrays, meta):
    src, tgt = net_names(meta)
    nets = _networks(t)
    for n in src + tgt:
        check_params(arrays, meta, n, [p.detach() for p in nets[n].parameters()],
                     tol=tols(meta)[1])


def _yield_losses(meta, closs, aloss, cpe):
    out = [float(closs[0])] + ([float(closs[1])] if meta["twin"] else [])
    out.append(None if aloss is None else float(aloss[1]))
    if cpe is not None:
        out += [float(cpe[0]), float(cpe[1])]
    return out


@pytest.mark.parametrize("name", CRR_CASES)
def test_generator_path_matches_reference(name):
    from reagent_b200.training import run_update

    arrays, meta = G.load(name)
    t = build_trainer(arrays, meta)
    batch = rlt_batch(arrays)
    opts = t.optimizers()
    assert len(opts) == meta["n_yields"]
    for it in range(meta["n_updates"]):
        inject_noise(t, arrays, meta, it)
        if it == 0:
            # drive the generator by hand to look at every gradient before its Adam step
            owners = [_networks(t)[n] for n in meta["optimizers"]]
            losses = []
            for oi, opt in enumerate(opts):
                loss = t.training_step(batch, it, oi)
                if oi < len(owners):
                    assert loss.grad_fn is not None
                    check_grads(arrays, meta, oi, t.net_grads(owners[oi]), tol=tols(meta)[0])
                    losses.append(loss)
                opt.zero_grad()
                loss.backward()
                opt.step()
            assert G.rel_err(t._ws["weight"], arrays["weight0"]) < tols(meta)[0]
        else:
            losses = run_update(t, batch, it)[:-1]
        check_losses(arrays, it, losses, tol=tols(meta)[0])
    _final_check(t, arrays, meta)


@pytest.mark.parametrize("name", CRR_CASES)
def test_train_batch_matches_reference_and_the_generator_bit_for_bit(name):
    from reagent_b200.training import run_update

    arrays, meta = G.load(name)
    fast, slow = build_trainer(arrays, meta), build_trainer(arrays, meta)
    batch = rlt_batch(arrays)
    for it in range(meta["n_updates"]):
        inject_noise(fast, arrays, meta, it)
        inject_noise(slow, arrays, meta, it)
        closs, aloss = fast.train_batch(batch, it)
        got = _yield_losses(meta, closs, aloss, getattr(fast, "cpe_losses", None))
        check_losses(arrays, it, got, tol=tols(meta)[0])
        gen = [None if l is None else float(l) for l in run_update(slow, batch, it)[:-1]]
        assert gen == got, (it, gen, got)
    _final_check(fast, arrays, meta)
    for a, b in zip(fast.parameters(), slow.parameters()):
        assert torch.equal(a, b)
    assert fast.all_batches_processed == slow.all_batches_processed == meta["n_updates"]


def test_cartpole_configuration_builds_through_the_manager_and_matches_reference():
    """reagent/gym/tests/configs/cartpole/discrete_crr_cartpole_online.yaml as written."""
    from reagent_b200.core.parameters import (EvaluationParameters, NormalizationData,
                                              NormalizationKey, NormalizationParameters,
                                              RLParameters)
    from reagent_b200.gym.policies import ActorPolicyWrapper
    from reagent_b200.model_managers import DiscreteCRR
    from reagent_b200.net_builder import DiscreteActorFullyConnected, FullyConnected
    from reagent_b200.core import types as rlt

    arrays, meta = G.load("crr_cartpole_manager")
    manager = DiscreteCRR(
        actions=["0", "1"], rl=RLParameters(gamma=0.99, target_update_rate=0.2, temperature=0.1),
        double_q_learning=True, delayed_policy_update=1,
        actor_net_builder=DiscreteActorFullyConnected(
            sizes=[1024, 1024], activations=["relu", "relu"], exploration_variance=1e-7),
        critic_net_builder=FullyConnected(sizes=[1024, 1024], activations=["relu", "relu"]),
        eval_parameters=EvaluationParameters(calc_cpe_in_training=False))
    norm = {NormalizationKey.STATE: NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS", mean=0.0, stddev=1.0)
        for i in range(4)})}
    t = manager.build_trainer(norm, use_gpu=True)
    assert t.actor_network.exploration_variance == 1e-7 and t.q2_network is not None
    for name, net in _networks(t).items():
        if net is not None:
            _load(arrays, meta, name, net)
    batch = rlt_batch(arrays)
    for it in range(meta["n_updates"]):
        inject_noise(t, arrays, meta, it)
        closs, aloss = t.train_batch(batch, it)
        check_losses(arrays, it, _yield_losses(meta, closs, aloss, None), tol=tols(meta)[0])
    _final_check(t, arrays, meta)
    policy = manager.create_policy(t)
    assert isinstance(policy, ActorPolicyWrapper)
    out = policy.act(rlt.FeatureData(batch.state.float_features[:5]))
    assert out.action.shape == (5, 2) and bool((out.action.abs() <= 1).all())
    # its own noise, drawn on the device: finite losses, parameters that keep moving
    t.noise_hook = None
    before = [p.detach().clone() for p in t.actor_network.parameters()]
    closs, aloss = t.train_batch(batch, 3)
    assert torch.isfinite(closs).all() and torch.isfinite(aloss).all()
    assert any(not torch.equal(a, b) for a, b in zip(before, t.actor_network.parameters()))


def test_validation_step_returns_the_three_losses_without_touching_anything():
    arrays, meta = G.load("crr_entropy_clip")
    t = build_trainer(arrays, meta)
    batch = rlt_batch(arrays)
    before = [p.detach().clone() for p in t.parameters()]
    without_reg, actor_loss, td_loss = t.validation_step(batch, 0)
    ref = arrays["losses"][0]  # update 0 sees the same parameters
    assert abs(float(td_loss) - ref[0]) <= 1e-5 * max(1.0, abs(ref[0]))
    assert float(without_reg) != float(actor_loss)  # the entropy term is on
    assert t._logged["eval_td_loss"] is td_loss
    assert all(torch.equal(a, b) for a, b in zip(before, t.parameters()))
    assert t.get_detached_model_outputs(batch.state)[1] is None
    t.strict_input_checks = True
    bad = rlt_batch(arrays)
    bad.extras.action_probability[3] = 0.0
    with pytest.raises(AssertionError, match="Logged action probability"):
        t.validation_step(bad, 0)


# ---------------------------------------------------------------------------
# FusedDqnStep
# ---------------------------------------------------------------------------
S, A, B, CAP = 6, 3, 128, 2048


def _stream(n, seed):
    rng = np.random.RandomState(seed)
    return dict(observation=rng.standard_normal((n, S)).astype(np.float32),
                action=rng.randint(0, A, n).astype(np.int64),
                reward=rng.standard_normal(n).astype(np.float32),
                terminal=rng.rand(n) < 0.02, priority=rng.uniform(0.1, 10.0, n))


def _setup(prioritized, exploration_variance=None, delayed=1):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import DuelingQNetwork, FullyConnectedActor
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, ReplayBuffer
    from reagent_b200.training import DiscreteCRRTrainer

    dev = torch.device("cuda", 0)
    data = _stream(CAP - 7, 3)
    if prioritized:
        rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAP, batch_size=B, device=dev)
    else:
        rb = ReplayBuffer(stack_size=1, replay_capacity=CAP, batch_size=B, device=dev)
        data.pop("priority")
    rb.add_batch(**data)
    torch.manual_seed(1)
    actor = FullyConnectedActor(S, A, [32, 16], ["relu", "relu"],
                                exploration_variance=exploration_variance).to(dev)
    q1 = DuelingQNetwork.make_fully_connected(S, A, [32, 16], ["relu", "relu"]).to(dev)
    q2 = DuelingQNetwork.make_fully_connected(S, A, [32, 16], ["relu", "relu"]).to(dev)
    t = DiscreteCRRTrainer(
        actor_network=actor, actor_network_target=actor.get_target_network(), q1_network=q1,
        q1_network_target=q1.get_target_network(), reward_network=None, q2_network=q2,
        q2_network_target=q2.get_target_network(),
        evaluation=EvaluationParameters(calc_cpe_in_training=False),
        rl=RLParameters(gamma=0.9, target_update_rate=0.05),
        q_network_optimizer=Optimizer__Union.default(lr=1e-2),
        actor_network_optimizer=Optimizer__Union.default(lr=1e-2),
        actions=[str(i) for i in range(A)], delayed_policy_update=delayed).to(dev)
    return rb, t


def _seed():
    random.seed(7)
    torch.manual_seed(7)
    np.random.seed(7)


@pytest.mark.parametrize("prefetch", [False, True])
def test_fused_step_with_host_rng_matches_the_hand_rolled_loop(prefetch):
    from reagent_b200.training.fused_step import FusedDqnStep

    n = 6
    rb, t = _setup(False)
    _seed()
    eager = []
    for _ in range(n + 1):  # the constructor runs one warm-up update
        eager.append(float(t.train_batch(rb.sample_discrete_dqn_batch(B, A))[0][0]))
    rb2, t2 = _setup(False)
    _seed()
    fused = FusedDqnStep(t2, rb2, B, prefetch=prefetch)
    got = []
    for _ in range(n):
        lh = fused.step()
        torch.cuda.synchronize()
        got.append(float(lh[0]))
    assert got == eager[1:], (got, eager[1:])
    for a, b in zip(t.parameters(), t2.parameters()):
        assert torch.equal(a, b)


def test_captured_online_step_matches_the_eager_one():
    """rng="device", online=True on the prioritized buffer: the captured step and the same step
    run eagerly agree bit for bit."""
    from reagent_b200.training.fused_step import FusedDqnStep

    def setup():
        rb, t = _setup(True)
        random.seed(5)
        return FusedDqnStep(t, rb, B, rng="device", online=True), None

    assert_captured_equals_eager(setup, _stream(12, 11), 12, lambda f: params(f.trainer))


def test_captured_online_step_draws_its_exploration_noise_inside_the_graph():
    from reagent_b200.training.fused_step import FusedDqnStep

    extra = _stream(8, 11)
    rb, t = _setup(True, exploration_variance=0.5)
    random.seed(5)
    fused = FusedDqnStep(t, rb, B, rng="device", online=True, slots=1)
    # the same transition and, with slots=1, the same graph: what differs between two replays
    # is the draw of the batch and the noise
    snap = [p.detach().clone() for p in t.actor_network.parameters()]
    losses = []
    for i in range(8):
        lh = fused.step({k: v[i] for k, v in extra.items()})
        torch.cuda.current_stream().synchronize()
        losses.append(float(lh[0]))
    fused.dr.raise_if_failed()
    assert all(np.isfinite(losses)) and len(set(losses)) == len(losses)
    assert any(not torch.equal(a, b) for a, b in zip(snap, t.actor_network.parameters()))
    assert all(torch.isfinite(p).all() for p in t.parameters())


def test_fused_step_refusals():
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    rb, t = _setup(True)
    with pytest.raises(NotImplementedError, match="importance weights"):
        FusedDqnStep(t, rb, B, rng="device", online=True, per=PrioritizedUpdate())
    with pytest.raises(NotImplementedError, match="single-GPU"):
        FusedDqnStep(t, rb, B, shard=(0, 2))
    with pytest.raises(NotImplementedError, match="single-GPU"):
        FusedDqnStep(t, rb, B, process_group=object())
    rb, t = _setup(True, delayed=2)
    with pytest.raises(NotImplementedError, match="delayed_policy_update"):
        FusedDqnStep(t, rb, B)
