"""GPU parity of ParametricDQNTrainer and C51Trainer (SURVEY.md 8f rank 3) against golden
vectors from the unmodified reference trainers (oracle/make_golden.py::pdqn_case / c51_case):
losses of every update, gradients of the first, parameters and targets after N updates."""
import pytest
import torch

from tests import golden_util as G
from tests.golden_cases import C51_CASES, PDQN_CASES

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _check_nets(pairs, arrays):
    for net, prefix in pairs:
        ps = list(net.parameters())
        want = G.net_pairs(arrays, prefix)
        assert len(ps) == 2 * len(want)
        for i, (w, b) in enumerate(want):
            assert G.rel_err(ps[2 * i], w) < TOL, (prefix, i)
            assert G.rel_err(ps[2 * i + 1], b) < TOL, (prefix, i)


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("name", PDQN_CASES)
def test_parametric_dqn_matches_reference(name, fast):
    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import ParametricDQNTrainer, run_update

    arrays, meta = G.load(name)
    S, AD = meta["S"], meta["AD"]
    q = FullyConnectedCritic(S, AD, meta["sizes"], meta["acts"])
    qt = q.get_target_network()
    G.load_into_module(arrays, "q0", q)
    G.load_into_module(arrays, "qt0", qt)
    rn = None
    if meta["with_reward_net"]:
        rn = FullyConnectedCritic(S, AD, meta["sizes"], meta["acts"])
        G.load_into_module(arrays, "r0", rn)
        rn = rn.cuda()
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"], q_network_loss=meta["loss"],
                      maxq_learning=meta["maxq"], multi_steps=meta["multi_steps"])
    t = ParametricDQNTrainer(q.cuda(), qt.cuda(), rn, rl=rl, double_q_learning=meta["double_q"],
                             optimizer=Optimizer__Union.default(lr=meta["lr"])).cuda()
    b = G.batch_tensors(arrays, "cuda")
    batch = rlt.ParametricDqnInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
        reward=b["reward"], time_diff=b["time_diff"],
        step=b["step"] if meta["multi_steps"] is not None else None, not_terminal=b["not_terminal"],
        action=rlt.FeatureData(b["action"]), next_action=rlt.FeatureData(b["next_action"]),
        possible_actions=rlt.FeatureData(b["possible_actions"]),
        possible_actions_mask=b["possible_actions_mask"],
        possible_next_actions=rlt.FeatureData(b["possible_next_actions"]),
        possible_next_actions_mask=b["possible_next_actions_mask"], extras=rlt.ExtraData())
    assert len(t.configure_optimizers()) == (3 if rn is not None else 2)
    for it in range(meta["n_updates"]):
        want = arrays["losses"][it]
        if fast:
            td = float(t.train_batch(batch, it))
            rl_ = float(t._ws["r_loss"]) if rn is not None else None
        elif it == 0:
            opts = t.optimizers()
            l0 = t.training_step(batch, it, 0)
            for i, g in enumerate(t.q_network_grads()):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < TOL, f"grad {i}"
            opts[0].zero_grad(); l0.backward(); opts[0].step()
            td, rl_ = float(l0.detach()), None
            for k in range(1, len(opts)):
                lk = t.training_step(batch, it, k)
                opts[k].zero_grad(); lk.backward(); opts[k].step()
                if rn is not None and k == 1:
                    rl_ = float(lk.detach())
        else:
            out = run_update(t, batch, it)
            td, rl_ = float(out[0]), (float(out[1]) if rn is not None else None)
        assert abs(td - want[0]) <= TOL * max(1.0, abs(want[0])), (it, td, want[0])
        if rn is not None:
            assert abs(rl_ - want[1]) <= TOL * max(1.0, abs(want[1])), (it, rl_, want[1])
    _check_nets([(t.q_network, "qN"), (t.q_network_target, "qtN")]
                + ([(t.reward_network, "rN")] if rn is not None else []), arrays)


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("name", C51_CASES)
def test_c51_matches_reference(name, fast):
    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import C51Trainer, run_update

    arrays, meta = G.load(name)
    S, A, N = meta["S"], meta["A"], meta["N"]
    dist = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"], num_atoms=N)
    G.load_into_module(arrays, "q0", dist)
    q = CategoricalDQN(dist, qmin=meta["qmin"], qmax=meta["qmax"], num_atoms=N)
    qt = q.get_target_network()
    G.load_into_module(arrays, "qt0", qt.distributional_network)
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"], maxq_learning=meta["maxq"],
                      multi_steps=meta["multi_steps"], reward_boost=meta["boost"])
    t = C51Trainer(q.cuda(), qt.cuda(), actions=[str(i) for i in range(A)], rl=rl,
                   double_q_learning=meta["double_q"], minibatch_size=meta["B"], num_atoms=N,
                   qmin=meta["qmin"], qmax=meta["qmax"],
                   optimizer=Optimizer__Union.default(lr=meta["lr"])).cuda()
    b = G.batch_tensors(arrays, "cuda")
    batch = rlt.DiscreteDqnInput(
        state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
        reward=b["reward"], time_diff=b["time_diff"],
        step=b["step"] if meta["multi_steps"] is not None else None, not_terminal=b["not_terminal"],
        action=b["action"], next_action=b["next_action"],
        possible_actions_mask=b["possible_actions_mask"],
        possible_next_actions_mask=b["possible_next_actions_mask"], extras=rlt.ExtraData())
    for it in range(meta["n_updates"]):
        want = arrays["losses"][it]
        if fast:
            loss = float(t.train_batch(batch, it))
        elif it == 0:
            opts = t.optimizers()
            l0 = t.training_step(batch, it, 0)
            for i, g in enumerate(t.q_network_grads()):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < TOL, f"grad {i}"
            opts[0].zero_grad(); l0.backward(); opts[0].step()
            l1 = t.training_step(batch, it, 1)
            opts[1].zero_grad(); l1.backward(); opts[1].step()
            loss = float(l0.detach())
        else:
            loss = float(run_update(t, batch, it)[0])
        assert abs(loss - want) <= TOL * max(1.0, abs(want)), (it, loss, want)
    _check_nets([(t.q_network.distributional_network, "qN"),
                 (t.q_network_target.distributional_network, "qtN")], arrays)
    # the model's own forward: expected values of the categorical distribution
    out = t.q_network(rlt.FeatureData(b["state"]))
    assert out.shape == (meta["B"], A)
