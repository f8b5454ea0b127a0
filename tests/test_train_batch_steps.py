"""`train_batch` steps every network through the trainer's map from a network to the optimizer
that trains it and to the target its Polyak update moves, built from configure_optimizers().
On the CPU: the maps against tables that restate, by hand, the optimizer index and the target of
each network's step.  On the GPU: `train_batch` against the generator under the Lightning-style
loop, bit for bit (DiscreteCRRTrainer has its own such test on its goldens)."""
import pytest
import torch

from tests.online_step import same_bits

S, A = 5, 3


def _dqn(cpe):
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import DQNTrainer

    q = FullyConnectedDQN(S, A, [8], ["relu"])
    ev = EvaluationParameters(calc_cpe_in_training=cpe)
    if not cpe:
        return DQNTrainer(q, q.get_target_network(), actions=["a", "b", "c"], evaluation=ev)
    r, c = FullyConnectedDQN(S, A, [8], ["relu"]), FullyConnectedDQN(S, A, [8], ["relu"])
    return DQNTrainer(q, q.get_target_network(), r, c, c.get_target_network(),
                      actions=["a", "b", "c"], evaluation=ev)


def _qrdqn():
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import QRDQNTrainer

    q = FullyConnectedDQN(S, A, [8], ["relu"], num_atoms=5)
    return QRDQNTrainer(q, q.get_target_network(), actions=["a", "b", "c"], num_atoms=5,
                        evaluation=EvaluationParameters(calc_cpe_in_training=False))


def _c51():
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.training import C51Trainer

    q = CategoricalDQN(FullyConnectedDQN(S, A, [8], ["relu"], num_atoms=5), qmin=-1.0, qmax=1.0,
                       num_atoms=5)
    return C51Trainer(q, q.get_target_network(), actions=["a", "b", "c"], num_atoms=5, qmin=-1.0,
                      qmax=1.0)


def _pdqn(reward):
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.training import ParametricDQNTrainer

    q = FullyConnectedCritic(S, A, [8], ["relu"])
    r = FullyConnectedCritic(S, A, [8], ["relu"]) if reward else None
    return ParametricDQNTrainer(q, q.get_target_network(), r)


def _bc():
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.training import BehavioralCloningTrainer

    return BehavioralCloningTrainer(FullyConnectedDQN(S, A, [8], ["relu"]))


def _crr(twin, cpe):
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import FullyConnectedActor, FullyConnectedDQN
    from reagent_b200.training import DiscreteCRRTrainer

    def net():
        return FullyConnectedDQN(S, A, [8], ["relu"])

    actor, q1 = FullyConnectedActor(S, A, [8], ["relu"]), net()
    q2 = net() if twin else None
    r, c = (net(), net()) if cpe else (None, None)
    return DiscreteCRRTrainer(
        actor_network=actor, actor_network_target=actor.get_target_network(), q1_network=q1,
        q1_network_target=q1.get_target_network(), reward_network=r, q2_network=q2,
        q2_network_target=None if q2 is None else q2.get_target_network(), q_network_cpe=c,
        q_network_cpe_target=None if c is None else c.get_target_network(),
        evaluation=EvaluationParameters(calc_cpe_in_training=cpe), double_q_learning=twin,
        actions=["a", "b", "c"])


def _sac(twin, alpha, value):
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.training import SACTrainer

    q2 = FullyConnectedCritic(S, 2, [8], ["relu"]) if twin else None
    v = FloatFeatureFullyConnected(S, 1, [8], ["relu"]) if value else None
    return SACTrainer(GaussianFullyConnectedActor(S, 2, [8], ["relu"]),
                      FullyConnectedCritic(S, 2, [8], ["relu"]), q2, v,
                      **({} if alpha else {"alpha_optimizer": None}))


def _td3(twin):
    from reagent_b200.models import FullyConnectedActor, FullyConnectedCritic
    from reagent_b200.training import TD3Trainer

    q2 = FullyConnectedCritic(S, 2, [8], ["relu"]) if twin else None
    return TD3Trainer(FullyConnectedActor(S, 2, [8], ["relu"]),
                      FullyConnectedCritic(S, 2, [8], ["relu"]), q2)


# (builder, [(network, index in optimizers(), target network or None)]) -- one row per Adam
CASES = {
    "dqn": (lambda: _dqn(False), [("q_network", 0, "q_network_target")]),
    "dqn_cpe": (lambda: _dqn(True), [("q_network", 0, "q_network_target"),
                                     ("reward_network", 1, None),
                                     ("q_network_cpe", 2, "q_network_cpe_target")]),
    "qrdqn": (_qrdqn, [("q_network", 0, "q_network_target")]),
    "c51": (_c51, [("q_network", 0, "q_network_target")]),
    "pdqn": (lambda: _pdqn(False), [("q_network", 0, "q_network_target")]),
    "pdqn_reward": (lambda: _pdqn(True), [("q_network", 0, "q_network_target"),
                                          ("reward_network", 1, None)]),
    "bc": (_bc, [("bc_net", 0, None)]),
    "crr_twin": (lambda: _crr(True, False), [("q1_network", 0, "q1_network_target"),
                                             ("q2_network", 1, "q2_network_target"),
                                             ("actor_network", 2, "actor_network_target")]),
    "crr_single": (lambda: _crr(False, False), [("q1_network", 0, "q1_network_target"),
                                                ("actor_network", 1, "actor_network_target")]),
    "crr_twin_cpe": (lambda: _crr(True, True), [("q1_network", 0, "q1_network_target"),
                                                ("q2_network", 1, "q2_network_target"),
                                                ("actor_network", 2, "actor_network_target"),
                                                ("reward_network", 3, None),
                                                ("q_network_cpe", 4, "q_network_cpe_target")]),
    "crr_single_cpe": (lambda: _crr(False, True), [("q1_network", 0, "q1_network_target"),
                                                   ("actor_network", 1, "actor_network_target"),
                                                   ("reward_network", 2, None),
                                                   ("q_network_cpe", 3, "q_network_cpe_target")]),
    "sac_twin_alpha": (lambda: _sac(True, True, False), [("q1_network", 0, "q1_network_target"),
                                                         ("q2_network", 1, "q2_network_target"),
                                                         ("actor_network", 2, None),
                                                         ("log_alpha", 3, None)]),
    "sac_twin": (lambda: _sac(True, False, False), [("q1_network", 0, "q1_network_target"),
                                                    ("q2_network", 1, "q2_network_target"),
                                                    ("actor_network", 2, None)]),
    "sac_single_alpha": (lambda: _sac(False, True, False), [("q1_network", 0, "q1_network_target"),
                                                            ("actor_network", 1, None),
                                                            ("log_alpha", 2, None)]),
    "sac_single": (lambda: _sac(False, False, False), [("q1_network", 0, "q1_network_target"),
                                                       ("actor_network", 1, None)]),
    "sac_twin_alpha_value": (lambda: _sac(True, True, True), [
        ("q1_network", 0, None), ("q2_network", 1, None), ("actor_network", 2, None),
        ("log_alpha", 3, None), ("value_network", 4, "value_network_target")]),
    "sac_twin_value": (lambda: _sac(True, False, True), [
        ("q1_network", 0, None), ("q2_network", 1, None), ("actor_network", 2, None),
        ("value_network", 3, "value_network_target")]),
    "sac_single_alpha_value": (lambda: _sac(False, True, True), [
        ("q1_network", 0, None), ("actor_network", 1, None), ("log_alpha", 2, None),
        ("value_network", 3, "value_network_target")]),
    "sac_single_value": (lambda: _sac(False, False, True), [
        ("q1_network", 0, None), ("actor_network", 1, None),
        ("value_network", 2, "value_network_target")]),
    "td3_twin": (lambda: _td3(True), [("q1_network", 0, "q1_network_target"),
                                      ("q2_network", 1, "q2_network_target"),
                                      ("actor_network", 2, "actor_network_target")]),
    "td3_single": (lambda: _td3(False), [("q1_network", 0, "q1_network_target"),
                                         ("actor_network", 1, "actor_network_target")]),
}


def _arena(trainer, name):
    x = getattr(trainer, name)
    return x._rb200_arena if isinstance(x, torch.nn.Parameter) else x.arena


@pytest.mark.parametrize("name", list(CASES))
def test_each_network_steps_its_own_optimizer_and_target(name):
    from reagent_b200.optimizer import FusedAdam

    build, rows = CASES[name]
    t = build()
    opts = t.optimizers()
    assert sum(isinstance(o, FusedAdam) for o in opts) == len(rows)
    for net, i, target in rows:
        arena = _arena(t, net)
        assert t.optimizer_of(arena) is opts[i], net
        pair = t._polyak_of.get(arena)
        if target is None:
            assert pair is None, net
        else:
            assert pair[0] is _arena(t, target), net
            assert pair[1].param_groups[0]["tau"] == t.tau
    assert len(t._polyak_of) == sum(target is not None for _, _, target in rows)
    with pytest.raises(KeyError):
        t.optimizer_of(object())


def _batch(name, it, B=64):
    """Seeded batch `it` of the input type of case `name`, on the GPU."""
    from reagent_b200.core import types as rlt

    gen = torch.Generator().manual_seed(100 + it)

    def rnd(*shape):
        return torch.randn(*shape, generator=gen).cuda()

    def onehot():
        return torch.nn.functional.one_hot(torch.randint(A, (B,), generator=gen), A).float().cuda()

    state, next_state, reward = rnd(B, S), rnd(B, S), rnd(B, 1)
    not_terminal = (torch.rand(B, 1, generator=gen) > 0.1).float().cuda()
    ones = torch.ones(B, A, device="cuda")
    if name == "bc":
        return rlt.BehavioralCloningModelInput(rlt.FeatureData(state), onehot(), ones)
    if name.startswith("td3"):
        return rlt.PolicyNetworkInput(
            state=rlt.FeatureData(state), next_state=rlt.FeatureData(next_state),
            action=rlt.FeatureData(rnd(B, 2).tanh()), next_action=rlt.FeatureData(rnd(B, 2).tanh()),
            reward=reward, not_terminal=not_terminal, step=None, time_diff=None,
            extras=rlt.ExtraData())
    if name.startswith("pdqn"):
        tiled = rlt.FeatureData(torch.eye(A, device="cuda").repeat(B, 1))
        return rlt.ParametricDqnInput(
            state=rlt.FeatureData(state), next_state=rlt.FeatureData(next_state), reward=reward,
            time_diff=torch.ones_like(reward), step=None, not_terminal=not_terminal,
            action=rlt.FeatureData(onehot()), next_action=rlt.FeatureData(onehot()),
            possible_actions=tiled, possible_actions_mask=ones, possible_next_actions=tiled,
            possible_next_actions_mask=ones, extras=rlt.ExtraData())
    return rlt.DiscreteDqnInput(
        state=rlt.FeatureData(state), next_state=rlt.FeatureData(next_state), reward=reward,
        time_diff=torch.ones_like(reward), step=None, not_terminal=not_terminal, action=onehot(),
        next_action=onehot(), possible_actions_mask=ones, possible_next_actions_mask=ones,
        extras=rlt.ExtraData(action_probability=torch.ones_like(reward)))


def _state(t):
    """Every parameter and buffer (targets included) and every Adam moment and step count."""
    from reagent_b200.optimizer import FusedAdam

    out = [v.detach().clone() for v in t.state_dict().values() if isinstance(v, torch.Tensor)]
    for o in t.optimizers():
        if isinstance(o, FusedAdam):
            out += [o.exp_avg.clone(), o.exp_avg_sq.clone(), o.step_t.clone()]
    return out


# TD3 trains its actor and moves every target on even batches only: 4 updates cover both phases
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dqn", "dqn_cpe", "qrdqn", "c51", "pdqn", "pdqn_reward", "bc",
                                  "td3_twin", "td3_single"])
def test_train_batch_matches_the_generator_bit_for_bit(name):
    from reagent_b200.training import run_update

    build = CASES[name][0]
    torch.manual_seed(0)
    fast = build().cuda()
    torch.manual_seed(0)
    slow = build().cuda()
    assert same_bits(_state(fast), _state(slow))
    for it in range(4):
        batch = _batch(name, it)
        for t in (fast, slow):
            t.noise_hook = lambda kind, shape, device, it=it: torch.randn(
                shape, generator=torch.Generator().manual_seed(10 * it + len(kind))).to(device)
        out = fast.train_batch(batch, it)
        got = (out[0] if name.startswith("td3") else out).reshape(-1)[0]
        want = run_update(slow, batch, it)[0]
        assert same_bits(got.reshape(()), want.detach().reshape(())), it
        assert same_bits(_state(fast), _state(slow)), it
    assert fast.all_batches_processed == slow.all_batches_processed == 4
