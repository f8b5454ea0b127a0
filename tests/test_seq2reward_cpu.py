"""Seq2Reward without a GPU: the oracle's internal consistency, gen_permutations, the parameter
and builder defaults, the library's shape refusals, and the host checks of valid_step and
all_permut."""
import pytest
import torch

from oracle import seq2reward_oracle as O
from oracle.mdnrnn_oracle import sample
from tests import seq2reward_cases as C
from tests.golden_util import grad_close, load, rel_err
from reagent_b200 import _lib
from reagent_b200.core import types as rlt
from reagent_b200.core.parameters import Seq2RewardTrainerParameters
from reagent_b200.model_managers import Seq2RewardModel
from reagent_b200.models import Seq2RewardNetwork
from reagent_b200.net_builder import Seq2RewardNetBuilder, ValueFullyConnected
from reagent_b200.training import Seq2RewardTrainer, gen_permutations, get_Q


def test_parameter_and_builder_defaults():
    p = Seq2RewardTrainerParameters()
    assert (p.learning_rate, p.multi_steps, p.action_names, p.compress_model_learning_rate,
            p.gamma, p.view_q_value, p.step_predict_net_size, p.reward_boost) == (
        0.001, 1, [], 0.001, 1.0, False, 64, None)
    b = Seq2RewardNetBuilder()
    assert (b.action_dim, b.num_hiddens, b.num_hidden_layers) == (2, 64, 2)
    m = Seq2RewardModel()
    assert isinstance(m.net_builder, Seq2RewardNetBuilder)
    assert isinstance(m.compress_net_builder, ValueFullyConnected)


@pytest.mark.parametrize("k,A", [(1, 6), (2, 3), (3, 2), (6, 2), (4, 3)])
def test_gen_permutations_lexical_one_hot(k, A):
    p = gen_permutations(k, A)
    assert p.shape == (k, A ** k, A)
    idx = p.argmax(dim=2).T.tolist()
    assert [tuple(r) for r in idx] == O.permutations(k, A)
    assert torch.all(p.sum(dim=2) == 1)


def test_network_keys_order():
    net = Seq2RewardNetwork(3, 2, 8, 2)
    keys = list(net.state_dict().keys())
    assert keys[:8] == ["rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0", "rnn.bias_hh_l0",
                        "rnn.weight_ih_l1", "rnn.weight_hh_l1", "rnn.bias_ih_l1", "rnn.bias_hh_l1"]
    assert keys[8:] == ["lstm_linear.weight", "lstm_linear.bias", "map_linear.weight",
                        "map_linear.bias"]
    flat = net.arena.flat
    assert all(p.data_ptr() >= flat.data_ptr() for p in net.parameters())


@pytest.mark.parametrize("shape", [(0, 2, 64, 2, 1), (257, 2, 64, 2, 1), (2, 17, 64, 2, 1),
                                   (2, 2, 129, 2, 1), (2, 2, 64, 5, 1), (2, 2, 64, 2, 17),
                                   (2, 4, 64, 2, 9), (2, 2, 64, 2, 0), (253, 2, 128, 4, 1),
                                   (256, 2, 128, 4, 1)])
def test_shape_refusals(shape):
    assert _lib.lib().rb200_seq2reward_check_shape(*shape) == _lib.E_INVALID
    assert "unsupported shape" in _lib.lib().rb200_last_error().decode()


def test_limits_accepted_and_workspace_arithmetic():
    lib = _lib.lib()
    assert lib.rb200_seq2reward_check_shape(252, 16, 128, 4, 4) == 0
    assert lib.rb200_seq2reward_check_shape(256, 16, 127, 4, 4) == 0
    assert lib.rb200_seq2reward_check_shape(256, 16, 128, 3, 4) == 0
    assert lib.rb200_seq2reward_check_shape(2, 2, 64, 2, 16) == 0
    # A 2, k 6, B 1024, H 64, L 2: 1024 * 2 ** 5 nodes of L * 2 * H floats
    assert lib.rb200_seq2reward_plan_workspace_bytes(1024, 2, 6, 64, 2) == 1024 * 32 * 256 * 4
    assert lib.rb200_seq2reward_plan_workspace_bytes(7, 6, 1, 64, 2) == 0
    cap = _lib.SEQ2REWARD_PLAN_BUDGET_BYTES
    assert lib.rb200_seq2reward_plan_workspace_bytes(100_000, 4, 8, 128, 4) <= cap


def test_oracle_q_is_the_max_of_the_forward():
    params = [p.double() for p in O.initial_params(0, 2, 3, 6, 2)]
    state = torch.randn(4, 2, dtype=torch.float64)
    q_all = O.get_q_all(params, state, 3, 3, 2)
    for j in range(1, 4):
        for b in range(4):
            for a in range(3):
                best = max(float(O.forward(params, state[b:b + 1], torch.nn.functional.one_hot(
                    torch.tensor([[x] for x in seq]), 3).double(), 2))
                    for seq in O.permutations(j, 3) if seq[0] == a)
                assert abs(float(q_all[b, j - 1, a]) - best) < 1e-12


def test_oracle_target_accumulates_in_fp64():
    r = torch.tensor([[1.0], *[[1e-8]] * 10])
    t = O.target(r, torch.tensor([11]), 1.0)
    assert t.float().item() == torch.cumsum(r, 0)[-1].item()
    assert t.float().item() != 1.0


def _trainer(k=3):
    params = Seq2RewardTrainerParameters(multi_steps=k, action_names=["0", "1"])
    return Seq2RewardTrainer(Seq2RewardNetwork(2, 2, 8, 1), params)


@pytest.mark.parametrize("valid", [[0, 1], [1, 4], [2, 6]])
def test_valid_step_host_check(valid):
    tr = _trainer(3)
    T, B = 5, 2
    b = rlt.MemoryNetworkInput(
        state=rlt.FeatureData(torch.zeros(T, B, 2)), next_state=rlt.FeatureData(torch.zeros(T, B, 2)),
        action=rlt.FeatureData(torch.zeros(T, B, 2)), reward=torch.zeros(T, B),
        not_terminal=torch.ones(T, B), time_diff=None, step=None,
        valid_step=torch.tensor(valid).unsqueeze(1))
    with pytest.raises(ValueError, match="valid_step"):
        tr._check_valid_step(b)


def test_all_permut_check():
    net = Seq2RewardNetwork(2, 2, 8, 1)
    bad = gen_permutations(3, 2).flip(1)
    with pytest.raises(ValueError, match="gen_permutations"):
        get_Q(net, torch.zeros(1, 2), bad)
    with pytest.raises(ValueError):
        get_Q(net, torch.zeros(1, 2), gen_permutations(3, 2)[0])
    # a valid tensor passes the check and then needs the GPU
    with pytest.raises(_lib.Rb200Error):
        get_Q(net, torch.zeros(1, 2), gen_permutations(3, 2))


@pytest.mark.parametrize("name", C.TRAINER_CASES)
def test_oracle_matches_trainer_golden(name):
    """The seeded networks are the reference's (SHA-256), and the fp64 oracle reproduces the
    reference's forward, both losses and the gradients of update 0."""
    arrays, meta = load(name)
    tr = C.build_trainer(arrays, meta, "cpu")
    p = [q.detach().double().requires_grad_(True) for q in tr.seq2reward_network.parameters()]
    sp = [q.detach().double().requires_grad_(True) for q in tr.step_predict_network.parameters()]
    b = C.batch(arrays, 0, "cpu")
    s0, act = b.state.float_features[0].double(), b.action.float_features.double()
    v = b.valid_step.flatten()
    out = O.forward(p, s0, act, meta["L"], v)
    n = arrays["out.acc_reward"].shape[0]
    assert rel_err(out[:n].detach(), arrays["out.acc_reward"]) < 1e-5
    mse = O.mse_loss(p, s0, act, b.reward, v, meta["L"], meta["gamma"])
    step = O.step_loss(sp, s0, v)
    assert abs(float(mse) - float(arrays["loss.mse"])) <= 1e-5 * max(1.0, float(arrays["loss.mse"]))
    assert abs(float(step) - float(arrays["loss.step"])) <= 1e-5 * max(1.0, float(arrays["loss.step"]))
    assert abs(float(mse) - arrays["losses"][0][0]) <= 1e-5 * max(1.0, arrays["losses"][0][0])
    for i, g in enumerate(O.grads(mse, p)):
        grad_close(sample(g), arrays[f"grad.{i}"], f"{name} grad.{i}")
    for i, g in enumerate(O.grads(step, sp)):
        grad_close(sample(g), arrays[f"sgrad.{i}"], f"{name} sgrad.{i}")


@pytest.mark.parametrize("name", C.PLAN_CASES)
def test_oracle_matches_plan_golden(name):
    arrays, meta = load(name)
    net = C.plan_network(arrays, meta, "cpu")
    p = [q.detach().double() for q in net.parameters()]
    state = torch.from_numpy(arrays["state"]).double()
    q_all = O.get_q_all(p, state, meta["A"], meta["k"], meta["L"])
    assert rel_err(q_all, arrays["q_all"]) < 1e-5
    assert rel_err(q_all[:, -1], arrays["q"]) < 1e-5
    assert torch.equal(gen_permutations(meta["k"], meta["A"]),
                       torch.from_numpy(arrays["permutations"]))


@pytest.mark.parametrize("name", C.COMPRESS_CASES)
def test_oracle_matches_compress_golden(name):
    arrays, meta = load(name)
    tr, net = C.build_compress(arrays, meta, "cpu")
    p = [q.detach().double() for q in net.parameters()]
    b = C.batch(arrays, 0, "cpu")
    s0 = b.state.float_features[0]
    q = O.get_q(p, s0.double(), meta["A"], meta["k"], meta["L"])
    assert rel_err(q, arrays["q"]) < 1e-5
    cp = [w.detach().double() for w in tr.compress_model_network.parameters()]
    out = O.mlp(cp, s0.double(), ["relu"] * len(meta["sizes"]) + ["linear"])
    mse, acc = O.compress(out, torch.from_numpy(arrays["q"]).double())
    assert abs(float(mse) - float(arrays["loss.mse"])) <= 1e-5 * max(1.0, float(arrays["loss.mse"]))
    assert float(acc) == float(arrays["loss.accuracy"])
