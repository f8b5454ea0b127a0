"""MDN-RNN on the H100: the fused forward, losses, BPTT and weight gradients against the
reference's goldens and the fp64 oracle, the two training paths bit for bit, and the limits."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mdnrnn_oracle as mo  # noqa: E402
from tests.golden_util import _adam_close, grad_close, load, rel_err  # noqa: E402

from reagent_b200 import _lib  # noqa: E402
from reagent_b200.core import types as rlt  # noqa: E402
from reagent_b200.core.parameters import (MDNRNNTrainerParameters, NormalizationData,  # noqa: E402
                                          NormalizationKey, NormalizationParameters)
from reagent_b200.models import MemoryNetwork  # noqa: E402
from reagent_b200.training import MDNRNNTrainer  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = ["mdnrnn_cartpole_features", "mdnrnn_cem_cartpole", "mdnrnn_defaults_seq",
         "mdnrnn_fit_last_odd"]
FIELDS = ("mus", "sigmas", "logpi", "reward", "not_terminal", "last_step_lstm_hidden",
          "last_step_lstm_cell", "all_steps_lstm_hidden")


def _params_of(meta):
    return MDNRNNTrainerParameters(
        hidden_size=meta["H"], num_hidden_layers=meta["L"], learning_rate=meta["lr"],
        num_gaussians=meta["G"], reward_loss_weight=meta["reward_weight"],
        next_state_loss_weight=meta["next_state_weight"],
        not_terminal_loss_weight=meta["not_terminal_weight"],
        fit_only_one_next_step=meta["fit_only_one_next_step"], action_dim=meta["A"])


def _check_initial(net, arrays):
    """The seeded initial weights are the golden's, bit for bit (SHA-256 of each tensor)."""
    for i, p in enumerate(net.mdnrnn.parameters()):
        np.testing.assert_array_equal(mo.digest(p), arrays[f"p0.{i}.sha256"], err_msg=f"p0.{i}")


def _trainer(arrays, meta):
    torch.manual_seed(meta["seed"])
    net = MemoryNetwork(meta["S"], meta["A"], meta["H"], meta["L"], meta["G"]).cuda()
    _check_initial(net, arrays)
    return MDNRNNTrainer(net, _params_of(meta))


def _weights_close(net, arrays, meta, n_updates):
    """Weights after `n_updates` Adam steps on the golden's subsample of every tensor."""
    m = dict(meta, n_updates=n_updates)
    for i, p in enumerate(net.mdnrnn.parameters()):
        _adam_close(mo.sample(p.detach()), torch.from_numpy(arrays[f"p{n_updates}.{i}"]), m)


def _batch(arrays, it):
    g = lambda k: torch.from_numpy(arrays[f"batch{it}.{k}"]).cuda()  # noqa: E731
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(g("state")), next_state=rlt.FeatureData(g("next_state")),
        action=rlt.FeatureData(g("action")), reward=g("reward"), not_terminal=g("not_terminal"),
        time_diff=None, step=None)


def _generator_update(tr, batch, it):
    """The reference's loop: train_step_gen -> backward -> optimizer.step."""
    opt = tr.optimizers()[0]
    gen = tr.train_step_gen(batch, it)
    loss = next(gen)
    opt.zero_grad()
    loss.backward()
    opt.step()
    with pytest.raises(StopIteration):
        next(gen)
    return float(loss)


@pytest.mark.parametrize("name", CASES)
def test_golden_forward_loss_grads_updates(name):
    arrays, meta = load(name)
    tr = _trainer(arrays, meta)
    b0 = _batch(arrays, 0)
    out = tr.memory_network(b0.state, b0.action)
    n = arrays["out.mus"].shape[1]
    for f in FIELDS:
        assert rel_err(getattr(out, f)[:, :n], arrays[f"out.{f}"]) < 1e-5, f
    for key, sd in (("loss_sd", meta["S"]), ("loss", None)):
        ls = tr.get_loss(b0, sd)
        for k in mo.LOSS_KEYS:
            assert rel_err(ls[k], arrays[f"{key}.{k}"]) < 1e-5, (key, k)
    for it in range(meta["n_updates"]):
        loss = _generator_update(tr, _batch(arrays, it), it)
        assert abs(loss - arrays["losses"][it]) <= 1e-5 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            for i, g in enumerate(tr.mdnrnn_grads()):
                grad_close(mo.sample(g), arrays[f"grad.{i}"], f"{name} grad.{i}")
        _weights_close(tr.memory_network, arrays, meta, it + 1)


def _run(arrays, meta, fast: bool):
    tr = _trainer(arrays, meta)
    losses = []
    for it in range(meta["n_updates"]):
        b = _batch(arrays, it)
        if fast:
            losses.append(tr.train_batch(b, it).clone())
        else:
            _generator_update(tr, b, it)
            losses.append(tr._ws.loss.clone())
    torch.cuda.synchronize()
    return tr, losses


@pytest.mark.parametrize("name", ["mdnrnn_defaults_seq", "mdnrnn_fit_last_odd"])
def test_train_batch_matches_generator_and_repeats(name):
    arrays, meta = load(name)
    runs = [_run(arrays, meta, fast) for fast in (False, True, True)]
    ref_tr, ref_losses = runs[0]
    for tr, losses in runs[1:]:
        for a, b in zip(losses, ref_losses):
            assert torch.equal(a, b)
        for p, q in zip(tr.memory_network.parameters(), ref_tr.memory_network.parameters()):
            assert torch.equal(p, q)
        o1, o2 = tr.optimizers()[0], ref_tr.optimizers()[0]
        assert torch.equal(o1.exp_avg, o2.exp_avg) and torch.equal(o1.exp_avg_sq, o2.exp_avg_sq)


def _oracle_case(T, B, S=5, A=2, H=64, L=2, G=5, seed=0):
    torch.manual_seed(seed)
    net = MemoryNetwork(S, A, H, L, G)
    with torch.no_grad():
        for p in net.mdnrnn.parameters():
            p.mul_(1.5)
    P64 = [p.detach().double().clone().requires_grad_(True) for p in net.mdnrnn.parameters()]
    net = net.cuda()
    g = torch.Generator().manual_seed(seed + 1)
    b = dict(state=torch.randn(T, B, S, generator=g),
             action=torch.nn.functional.one_hot(torch.randint(A, (T, B), generator=g), A).float(),
             next_state=torch.randn(T, B, S, generator=g), reward=torch.randn(T, B, generator=g),
             not_terminal=(torch.rand(T, B, generator=g) > 0.2).float())
    return net, P64, b


@pytest.mark.parametrize("T", [1, 6, 16])
@pytest.mark.parametrize("B", [1, 15, 17, 1024])
def test_against_fp64_oracle(T, B):
    fit = T == 6
    net, P64, b = _oracle_case(T, B)
    params = MDNRNNTrainerParameters(fit_only_one_next_step=fit, not_terminal_loss_weight=3.0)
    tr = MDNRNNTrainer(net, params)
    cb = rlt.MemoryNetworkInput(
        state=rlt.FeatureData(b["state"].cuda()), next_state=rlt.FeatureData(b["next_state"].cuda()),
        action=rlt.FeatureData(b["action"].cuda()), reward=b["reward"].cuda(),
        not_terminal=b["not_terminal"].cuda(), time_diff=None, step=None)
    out = tr.memory_network(cb.state, cb.action)
    b64 = {k: v.double() for k, v in b.items()}
    ref = mo.forward(P64, b64["state"], b64["action"], 2, 5)
    for f in FIELDS:
        assert rel_err(getattr(out, f), ref[f].detach()) < 2e-5, f
    losses = next(tr.train_step_gen(cb, 0))
    ls = mo.losses(ref, b64["next_state"], b64["reward"], b64["not_terminal"],
                   not_terminal_weight=3.0, fit_only_one_next_step=fit, state_dim=5)
    assert rel_err(losses, ls["loss"].detach()) < 2e-5
    for k, v in zip(mo.LOSS_KEYS, tr._ws.loss):
        assert rel_err(v, ls[k].detach()) < 2e-5, k
    ls["loss"].backward()
    for i, (g, p) in enumerate(zip(tr.mdnrnn_grads(), P64)):
        grad_close(g, p.grad, f"T{T} B{B} grad.{i}", l2_tol=1e-4, max_tol=1e-3)


def test_shape_limits_on_gpu():
    # the largest shape: hidden 128, 4 layers, S + A = 256, (2S + 1) G + 2 = 803
    net, P64, b = _oracle_case(3, 20, S=200, A=56, H=128, L=4, G=2)
    tr = MDNRNNTrainer(net, MDNRNNTrainerParameters())
    cb = rlt.MemoryNetworkInput(
        state=rlt.FeatureData(b["state"].cuda()), next_state=rlt.FeatureData(b["next_state"].cuda()),
        action=rlt.FeatureData(b["action"].cuda()), reward=b["reward"].cuda(),
        not_terminal=b["not_terminal"].cuda(), time_diff=None, step=None)
    losses = tr.train_batch(cb)
    b64 = {k: v.double() for k, v in b.items()}
    ref = mo.losses(mo.forward(P64, b64["state"], b64["action"], 4, 2), b64["next_state"],
                    b64["reward"], b64["not_terminal"], state_dim=200)
    assert rel_err(losses[3], ref["loss"].detach()) < 2e-5
    big = MemoryNetwork(4, 2, 129, 2, 1).cuda()
    with pytest.raises(_lib.Rb200Error, match="unsupported shape"):
        big(rlt.FeatureData(torch.zeros(1, 4, 4, device="cuda")),
            rlt.FeatureData(torch.zeros(1, 4, 2, device="cuda")))


def test_world_model_manager_trains_to_golden():
    """configs/world_model/cartpole_features.yaml through WorldModel.build_trainer."""
    from reagent_b200.model_managers import WorldModel

    arrays, meta = load("mdnrnn_cartpole_features")
    manager = WorldModel(trainer_param=MDNRNNTrainerParameters(
        hidden_size=50, num_hidden_layers=2, learning_rate=0.001, not_terminal_loss_weight=1,
        next_state_loss_weight=1, reward_loss_weight=1, num_gaussians=1))
    norm = {NormalizationKey.STATE: NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS") for i in range(4)})}
    torch.manual_seed(meta["seed"])
    tr = manager.build_trainer(norm, use_gpu=True)
    _check_initial(tr.memory_network, arrays)
    for it in range(meta["n_updates"]):
        tr.train_batch(_batch(arrays, it), it)
    _weights_close(tr.memory_network, arrays, meta, meta["n_updates"])


@pytest.mark.parametrize("kind,num_actions", [("discrete", 3), ("continuous", None)])
def test_replay_buffer_to_train_batch(kind, num_actions):
    """Stacked ReplayBuffer -> MemoryNetworkInputMaker -> train_batch, on the reference's
    replay contents."""
    from reagent_b200.gym.preprocessors.trainer_preprocessor import MemoryNetworkInputMaker
    from reagent_b200.replay_memory.circular_replay_buffer import ReplayBuffer

    arrays, _ = load("memory_input_maker")
    adds = {k: arrays[f"{kind}.add.{k}"] for k in ("observation", "action", "reward", "terminal")}
    rb = ReplayBuffer(stack_size=3, replay_capacity=64, batch_size=8,
                      return_everything_as_stack=True)
    for i in range(len(adds["reward"])):
        rb.add(observation=adds["observation"][i], action=adds["action"][i],
               reward=adds["reward"][i], terminal=adds["terminal"][i])
    s = rb.sample_transition_batch(batch_size=8,
                                   indices=torch.from_numpy(arrays[f"{kind}.indices"]))
    for f in ("state", "action", "reward", "next_state", "terminal"):
        np.testing.assert_array_equal(getattr(s, f).cpu().numpy(), arrays[f"{kind}.sample.{f}"], f)
    s = type(s)(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in s._asdict().items()})
    batch = MemoryNetworkInputMaker(num_actions)(s)
    for f, v in (("state", batch.state.float_features), ("action", batch.action.float_features),
                 ("next_state", batch.next_state.float_features), ("reward", batch.reward),
                 ("not_terminal", batch.not_terminal)):
        np.testing.assert_array_equal(v.cpu().numpy(), arrays[f"{kind}.out.{f}"], f)
    A = batch.action.float_features.shape[2]
    torch.manual_seed(0)
    net = MemoryNetwork(4, A, 16, 2, 2)
    P64 = [p.detach().double().clone() for p in net.mdnrnn.parameters()]
    tr = MDNRNNTrainer(net.cuda(), MDNRNNTrainerParameters(action_dim=A))
    losses = tr.train_batch(batch)
    b64 = {k: torch.from_numpy(arrays[f"{kind}.out.{k}"]).double()
           for k in ("state", "action", "next_state", "reward", "not_terminal")}
    ref = mo.losses(mo.forward(P64, b64["state"], b64["action"], 2, 2), b64["next_state"],
                    b64["reward"], b64["not_terminal"], state_dim=4)
    assert rel_err(losses[3], ref["loss"]) < 2e-5
