"""Host-side API surface (no GPU): constructors, optimizer order, yield contract metadata,
loud failure without CUDA."""
import inspect
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_trainer_constructors_and_optimizer_order():
    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import EvaluationParameters
    from reagent_b200.models import (FullyConnectedActor, FullyConnectedCritic, FullyConnectedDQN,
                                     GaussianFullyConnectedActor)
    from reagent_b200.optimizer import FusedAdam, SoftUpdate
    from reagent_b200.training import DQNTrainer, QRDQNTrainer, SACTrainer, TD3Trainer

    ev = EvaluationParameters(calc_cpe_in_training=False)
    q = FullyConnectedDQN(8, 3, [16], ["relu"])
    t = DQNTrainer(q, q.get_target_network(), actions=["a", "b", "c"], evaluation=ev)
    assert [type(o) for o in t.optimizers()] == [FusedAdam, SoftUpdate]
    assert inspect.signature(t.train_step_gen).parameters["training_batch"].annotation is rlt.DiscreteDqnInput
    with pytest.raises(AssertionError, match="reward_network is required for CPE"):
        DQNTrainer(q, q.get_target_network(), actions=["a", "b", "c"])  # CPE on by default (as the reference)
    rn, qc = FullyConnectedDQN(8, 3, [16], ["relu"]), FullyConnectedDQN(8, 3, [16], ["relu"])
    tc = DQNTrainer(q, q.get_target_network(), rn, qc, qc.get_target_network(), actions=["a", "b", "c"])
    assert [type(o) for o in tc.optimizers()] == [FusedAdam, FusedAdam, FusedAdam, SoftUpdate]
    assert tc.metrics_to_score == ["reward"] and tc.reward_idx_offsets.tolist() == [0]
    qq = FullyConnectedDQN(8, 3, [16], ["relu"], num_atoms=5)
    tq = QRDQNTrainer(qq, qq.get_target_network(), actions=["a", "b", "c"], num_atoms=5, evaluation=ev)
    assert tq.quantiles.shape == (1, 5) and abs(float(tq.quantiles[0, 0]) - 0.1) < 1e-7
    c1, c2 = FullyConnectedCritic(8, 2, [16], ["relu"]), FullyConnectedCritic(8, 2, [16], ["relu"])
    ts = SACTrainer(GaussianFullyConnectedActor(8, 2, [16], ["relu"]), c1, c2)
    assert [type(o) for o in ts.optimizers()] == [FusedAdam] * 4 + [SoftUpdate]
    assert inspect.signature(ts.train_step_gen).parameters["training_batch"].annotation is rlt.PolicyNetworkInput
    ts2 = SACTrainer(GaussianFullyConnectedActor(8, 2, [16], ["relu"]), c1, None, alpha_optimizer=None)
    assert len(ts2.optimizers()) == 3
    tt = TD3Trainer(FullyConnectedActor(8, 2, [16], ["relu"]), c1, c2)
    assert [type(o) for o in tt.optimizers()] == [FusedAdam] * 3 + [SoftUpdate]


def test_state_dict_keys_match_reference_layout():
    from reagent_b200.models import FullyConnectedDQN

    q = FullyConnectedDQN(4, 2, [8, 6], ["relu", "tanh"])
    assert list(q.state_dict().keys()) == [
        "fc.dnn.0.0.weight", "fc.dnn.0.0.bias", "fc.dnn.1.0.weight", "fc.dnn.1.0.bias",
        "fc.dnn.2.0.weight", "fc.dnn.2.0.bias"]
    # parameters are views into one flat arena; deepcopy gets its own arena
    base = q.arena.flat.data_ptr()
    assert q.fc.dnn[0][0].weight.data_ptr() == base
    qt = q.get_target_network()
    assert qt.arena.flat.data_ptr() != base and torch.equal(qt.arena.flat, q.arena.flat)
    sd = {k: torch.randn_like(v) for k, v in q.state_dict().items()}
    q.load_state_dict(sd)
    assert torch.equal(q.fc.dnn[1][0].weight, sd["fc.dnn.1.0.weight"])
    assert q.fc.dnn[1][0].weight.data_ptr() != q.fc.dnn[0][0].weight.data_ptr()
    a = q.arena
    assert torch.equal(a.flat[a.w_off[1]: a.w_off[1] + 48].view(6, 8), sd["fc.dnn.1.0.weight"])


def test_no_cpu_fallback():
    from reagent_b200 import _lib
    from reagent_b200.core import types as rlt
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.preprocessing import Preprocessor
    from reagent_b200.core.parameters import NormalizationParameters as NP

    q = FullyConnectedDQN(4, 2, [8], ["relu"])
    with pytest.raises(_lib.Rb200Error):
        q(rlt.FeatureData(torch.randn(3, 4)))
    p = Preprocessor({1: NP("CONTINUOUS", mean=0.0, stddev=1.0)})
    with pytest.raises(_lib.Rb200Error):
        p(torch.randn(3, 1), torch.ones(3, 1))


def test_net_builders_and_managers_construct():
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters as NP
    from reagent_b200.net_builder import FullyConnected, GaussianFullyConnected, ParametricFullyConnected, Quantile

    s = NormalizationData({i: NP("CONTINUOUS", mean=0.0, stddev=1.0) for i in range(6)})
    a = NormalizationData({i: NP("CONTINUOUS_ACTION", min_value=-1.0, max_value=1.0) for i in range(2)})
    assert FullyConnected(sizes=[8], activations=["relu"]).build_q_network(None, s, 3).fc.layers == [6, 8, 3]
    assert Quantile(sizes=[8], activations=["relu"]).build_q_network(s, 3, 5).fc.layers == [6, 8, 15]
    assert ParametricFullyConnected().build_q_network(s, a).fc.layers == [8, 128, 64, 1]
    assert GaussianFullyConnected().build_actor(None, s, a).fc.layers == [6, 128, 64, 4]
    from reagent_b200.model_managers import DiscreteDQN
    m = DiscreteDQN(actions=["0", "1"])
    assert m.eval_parameters.calc_cpe_in_training  # the reference default (core/parameters.py:118-120)
    with pytest.raises(RuntimeError):
        m.build_trainer({"state": s}, use_gpu=False)


def test_input_makers_match_reference_formulas():
    import collections

    from reagent_b200.gym.preprocessors.trainer_preprocessor import (DiscreteDqnInputMaker,
                                                                    PolicyNetworkInputMaker)

    B = collections.namedtuple("b", ["state", "action", "reward", "next_state", "next_action", "terminal"])
    b = B(torch.randn(4, 3), torch.tensor([[0], [2], [1], [2]]), torch.randn(4, 1), torch.randn(4, 3),
          torch.tensor([[1], [0], [2], [1]]), torch.tensor([[False], [True], [False], [False]]))
    out = DiscreteDqnInputMaker(3)(b)
    assert out.action.tolist() == [[1, 0, 0], [0, 0, 1], [0, 1, 0], [0, 0, 1]]
    assert out.next_action.tolist() == [[0, 1, 0], [0, 0, 0], [0, 0, 1], [0, 1, 0]]
    assert out.not_terminal.reshape(-1).tolist() == [1, 0, 1, 1]
    bc = B(torch.randn(2, 3), torch.tensor([[0.0, 2.0], [1.0, -2.0]]), torch.randn(2, 1), torch.randn(2, 3),
           torch.tensor([[2.0, 2.0], [0.0, 0.0]]), torch.tensor([[True], [False]]))
    oc = PolicyNetworkInputMaker([-2.0, -2.0], [2.0, 2.0])(bc)
    assert oc.action.float_features.tolist() == [[0.0, 1.0], [0.5, -1.0]]
    assert oc.next_action.float_features.tolist() == [[0.0, 0.0], [0.0, 0.0]]


def test_dueling_network_layout_cpu():
    """DuelingQNetwork: reference sub-module names / state_dict keys; all parameters are views
    into one arena whose compute description is the equivalent plain MLP."""
    from reagent_b200.models import DuelingQNetwork
    from reagent_b200.net_builder import Dueling
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters as NP

    q = DuelingQNetwork.make_fully_connected(12, 5, [24, 16], ["relu", "tanh"])
    keys = list(q.state_dict().keys())
    assert keys == [f"{part}_network.fc.dnn.{i}.0.{w}" for part in ("shared", "advantage", "value")
                    for i in (0, 1) for w in ("weight", "bias")]
    ar = q.arena
    assert ar.dims == [12, 24, 16, 16, 5] and len(ar.acts) == 4
    base, end = ar.flat.data_ptr(), ar.flat.data_ptr() + 4 * ar.n_true
    for p in q.parameters():
        assert base <= p.data_ptr() < end, "every true parameter lives in the arena"
        assert p._rb200_arena is ar
    # the two first head layers are consecutive row blocks of the stacked [E x E] layer
    a0, v0 = q.advantage_network.fc.dnn[0][0].weight, q.value_network.fc.dnn[0][0].weight
    assert v0.data_ptr() - a0.data_ptr() == 4 * a0.numel()
    qt = q.get_target_network()
    assert qt.arena is not ar and torch.equal(qt.arena.flat[: ar.n_true], ar.flat[: ar.n_true])
    sd = {k: torch.randn_like(v) for k, v in q.state_dict().items()}
    q.load_state_dict(sd)
    assert torch.equal(ar.flat[ar.o_wa: ar.o_wa + 5 * 8].view(5, 8), sd["advantage_network.fc.dnn.1.0.weight"])
    with pytest.raises(AssertionError):
        DuelingQNetwork.make_fully_connected(12, 5, [24, 15], ["relu", "relu"])  # odd embedding
    s = NormalizationData({i: NP("CONTINUOUS", mean=0.0, stddev=1.0) for i in range(6)})
    net = Dueling(sizes=[8, 4], activations=["relu", "relu"]).build_q_network(None, s, 3)
    assert isinstance(net, DuelingQNetwork) and net.arena.dims == [6, 8, 4, 4, 3]
