"""Seq2Reward on the GPU: the forward, gradients, plan and compress head against the fp64
oracle (oracle/seq2reward_oracle.py), the plan bit for bit against the forward on the expanded
batch, the two training paths against each other, the manager, and a learning check."""
import numpy as np
import pytest
import torch

from oracle import seq2reward_oracle as O
from oracle.mdnrnn_oracle import sample
from tests import seq2reward_cases as C
from tests.golden_util import _adam_close, grad_close, load, rel_err
from reagent_b200.core import types as rlt
from reagent_b200.core.parameters import NormalizationData, NormalizationParameters, Seq2RewardTrainerParameters
from reagent_b200.models import FloatFeatureFullyConnected, Seq2RewardNetwork
from reagent_b200.training import (CompressModelTrainer, Seq2RewardTrainer, gen_permutations,
                                   get_Q, plan_short_sequence_q, run_update)

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _net(S, A, H, L, seed=0):
    torch.manual_seed(seed)
    return Seq2RewardNetwork(S, A, H, L).to(DEV)


def _params64(net):
    return [p.detach().cpu().double().requires_grad_(True) for p in net.parameters()]


def _batch(S, A, T, B, k, seed=0, device=DEV):
    g = torch.Generator().manual_seed(seed)
    state = torch.randn(T, B, S, generator=g)
    action = torch.nn.functional.one_hot(torch.randint(0, A, (T, B), generator=g), A).float()
    reward = torch.randn(T, B, generator=g)
    valid = torch.randint(1, min(T, k) + 1, (B,), generator=g)
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(state.to(device)), next_state=rlt.FeatureData(state.to(device)),
        action=rlt.FeatureData(action.to(device)), reward=reward.to(device),
        not_terminal=torch.ones(T, B, device=device), time_diff=None, step=None,
        valid_step=valid.to(device).unsqueeze(1))


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-12))


@pytest.mark.parametrize("T", [1, 6, 16])
@pytest.mark.parametrize("B", [1, 15, 17, 1024])
def test_forward_matches_oracle(T, B):
    S, A, H, L = 3, 2, 64, 2
    net = _net(S, A, H, L)
    b = _batch(S, A, T, B, T)
    p = _params64(net)
    for valid in (None, torch.ones(B, dtype=torch.long), torch.full((B,), T)):
        got = net(b.state, b.action, None if valid is None else valid.to(DEV)).acc_reward
        want = O.forward(p, b.state.float_features[0].cpu().double(),
                         b.action.float_features.cpu().double(), L, valid)
        assert got.shape == (B, 1)
        assert _rel(got, want) < 1e-5


@pytest.mark.parametrize("S,A,T,B,H,L,gamma", [(2, 2, 6, 1024, 64, 2, 1.0),
                                               (5, 3, 4, 37, 37, 1, 0.9),
                                               (3, 4, 3, 17, 128, 4, 0.5),
                                               (252, 16, 3, 17, 128, 4, 1.0),
                                               (256, 16, 3, 17, 127, 4, 1.0)])
def test_losses_and_grads_match_oracle(S, A, T, B, H, L, gamma):
    net = _net(S, A, H, L)
    k = T
    params = Seq2RewardTrainerParameters(multi_steps=k, action_names=[str(i) for i in range(A)],
                                         gamma=gamma)
    tr = Seq2RewardTrainer(net, params).to(DEV)
    b = _batch(S, A, T, B, k)
    mse, step = tr._step(b, train=True)
    p = _params64(net)
    sp = [q.detach().cpu().double().requires_grad_(True) for q in tr.step_predict_network.parameters()]
    s0 = b.state.float_features[0].cpu().double()
    act = b.action.float_features.cpu().double()
    v = b.valid_step.flatten().cpu()
    lo = O.mse_loss(p, s0, act, b.reward.cpu(), v, L, gamma)
    ls = O.step_loss(sp, s0, v)
    assert abs(float(mse) - float(lo.detach())) <= 1e-5 * max(1.0, abs(float(lo.detach())))
    assert abs(float(step) - float(ls.detach())) <= 1e-5 * max(1.0, abs(float(ls.detach())))
    tgt = O.target(b.reward.cpu(), v, gamma).squeeze(1)
    assert torch.equal(tr._ws.target.cpu(), tgt.float())
    for i, (g, w) in enumerate(zip(tr.seq2reward_grads(), O.grads(lo, p))):
        grad_close(g, w, f"grad.{i}")
    for i, (g, w) in enumerate(zip(tr.step_predict_grads(), O.grads(ls, sp))):
        grad_close(g, w, f"sgrad.{i}")


@pytest.mark.parametrize("S,A,k,H,L,B", [(2, 6, 1, 64, 2, 5), (2, 2, 3, 64, 2, 33),
                                         (2, 2, 6, 64, 2, 20), (3, 3, 4, 37, 1, 7),
                                         (4, 4, 3, 128, 4, 17), (1, 16, 2, 8, 1, 3)])
def test_plan_matches_oracle_and_forward(S, A, k, H, L, B):
    net = _net(S, A, H, L)
    g = torch.Generator().manual_seed(1)
    state = torch.randn(B, S, generator=g).to(DEV)
    q, q_all = net.plan(state, k, all_horizons=True)
    p = _params64(net)
    want = O.get_q_all(p, state.cpu().double(), A, k, L)
    assert _rel(q_all, want) < 1e-5
    assert torch.equal(q, q_all[:, -1])
    # bit for bit: the forward over the reference's expanded batch, at every horizon
    for j in range(1, k + 1):
        perm = gen_permutations(j, A).to(DEV)
        n = perm.shape[1]
        s = state.unsqueeze(0).repeat_interleave(n, dim=1)
        r = net(rlt.FeatureData(s), rlt.FeatureData(perm.repeat(1, B, 1))).acc_reward
        ref = r.reshape(B, A, n // A).max(dim=2).values
        assert torch.equal(q_all[:, j - 1], ref), j
        qj, _ = net.plan(state, j)
        assert torch.equal(qj, q_all[:, j - 1]), j
    assert torch.equal(get_Q(net, state, gen_permutations(k, A)), q)


def test_plan_chunks_the_states(monkeypatch):
    """A workspace smaller than the batch needs runs the walk in chunks, with the same result."""
    from reagent_b200 import _lib
    net = _net(2, 2, 64, 2)
    state = torch.randn(50, 2, device=DEV)
    q_full, qa_full = net.plan(state, 6, all_horizons=True)
    lib = _lib.lib()
    per = int(lib.rb200_seq2reward_plan_workspace_bytes(1, 2, 6, 64, 2))
    orig = _lib.lib

    class Small:
        def __getattr__(self, name):
            if name == "rb200_seq2reward_plan_workspace_bytes":
                return lambda *a: 7 * per
            return getattr(orig(), name)
    monkeypatch.setattr(_lib, "lib", lambda: Small())
    net._plan_ws.clear()
    q, qa = net.plan(state, 6, all_horizons=True)
    assert torch.equal(q, q_full) and torch.equal(qa, qa_full)


def test_short_sequence_planner():
    net = _net(2, 2, 16, 1)
    params = Seq2RewardTrainerParameters(multi_steps=4, action_names=["0", "1"])
    tr = Seq2RewardTrainer(net, params).to(DEV)
    state = torch.randn(9, 2, device=DEV)
    got = plan_short_sequence_q(net, tr.step_predict_network, state, 4, 2)
    prob = torch.softmax(tr.step_predict_network(state), dim=1)
    qs = torch.stack([get_Q(net, state, gen_permutations(s, 2)) for s in range(1, 5)], dim=1)
    assert torch.allclose(got, (qs * prob.unsqueeze(2)).sum(1), rtol=1e-6, atol=1e-6)


def test_train_batch_matches_train_step_gen_and_does_not_sync():
    S, A, T, B, H, L = 2, 2, 6, 256, 32, 2
    params = Seq2RewardTrainerParameters(learning_rate=0.005, multi_steps=6,
                                         action_names=["0", "1"], view_q_value=True)
    t1 = Seq2RewardTrainer(_net(S, A, H, L), params).to(DEV)
    t2 = Seq2RewardTrainer(_net(S, A, H, L), params).to(DEV)
    for a, c in zip(list(t1.parameters()), list(t2.parameters())):
        assert torch.equal(a, c)
    batches = [_batch(S, A, T, B, 6, seed=i) for i in range(3)]
    for i, b in enumerate(batches):
        t1.train_batch(b, i)
        run_update(t2, b, i)
    for a, c in zip(list(t1.parameters()), list(t2.parameters())):
        assert torch.equal(a, c)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t1.train_batch(batches[0])
        get_Q(t1.seq2reward_network, batches[0].state.float_features[0], t1.all_permut)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_valid_step_out_of_range_raises():
    params = Seq2RewardTrainerParameters(multi_steps=3, action_names=["0", "1"])
    tr = Seq2RewardTrainer(_net(2, 2, 8, 1), params).to(DEV)
    b = _batch(2, 2, 6, 8, 3)
    b.valid_step[0] = 4
    with pytest.raises(ValueError):
        next(tr.train_step_gen(b, 0))
    with pytest.raises(ValueError):
        tr.validation_step(b, 0)


def test_compress_head_and_ties():
    S, A, k, B = 2, 2, 6, 64
    net = _net(S, A, 16, 2)
    params = Seq2RewardTrainerParameters(multi_steps=k, action_names=["0", "1"])
    torch.manual_seed(3)
    comp = FloatFeatureFullyConnected(S, A, [8, 8], ["relu", "relu"]).to(DEV)
    tr = CompressModelTrainer(comp, net, params)
    b = _batch(S, A, k, B, k)
    loss = tr._step(b, train=True)
    s0 = b.state.float_features[0]
    q = O.get_q(_params64(net), s0.cpu().double(), A, k, 2)
    out = comp(rlt.FeatureData(s0)).cpu().double()
    mse, acc = O.compress(out, q)
    assert abs(float(loss[0]) - float(mse)) <= 1e-5 * max(1.0, float(mse))
    assert float(loss[1]) == float(acc)
    # every sequence ties once lstm_linear.weight is zero: q is constant, argmax is action 0
    with torch.no_grad():
        net.lstm_linear.weight.zero_()
    loss = tr._step(b, train=False)
    q = net.plan(s0, k)[0]
    assert torch.all(q == q[:, :1])
    want = (torch.argmax(comp(rlt.FeatureData(s0)), dim=1) == 0).float().mean()
    assert float(loss[1]) == float(want)


def _norm(n):
    return NormalizationData(dense_normalization_parameters={
        i: NormalizationParameters(feature_type="CONTINUOUS", mean=0.0, stddev=1.0)
        for i in range(n)})


def _game_batch(B, seed, device=DEV):
    """State: one-hot class c of 2.  Reward 1 at every step whose action is c; valid steps
    1..6.  So Q(s, c) = 6 and Q(s, other) = 5."""
    g = torch.Generator().manual_seed(seed)
    T = 6
    c = torch.randint(0, 2, (B,), generator=g)
    a = torch.randint(0, 2, (T, B), generator=g)
    state = torch.nn.functional.one_hot(c, 2).float().unsqueeze(0).repeat(T, 1, 1)
    reward = (a == c.unsqueeze(0)).float()
    valid = torch.randint(1, T + 1, (B,), generator=g)
    return rlt.MemoryNetworkInput(
        state=rlt.FeatureData(state.to(device)), next_state=rlt.FeatureData(state.to(device)),
        action=rlt.FeatureData(torch.nn.functional.one_hot(a, 2).float().to(device)),
        reward=reward.to(device), not_terminal=torch.ones(T, B, device=device), time_diff=None,
        step=None, valid_step=valid.unsqueeze(1).to(device))


def test_manager_learns_and_compress_distils():
    from reagent_b200.model_managers import Seq2RewardModel
    torch.manual_seed(0)
    mgr = Seq2RewardModel(trainer_param=Seq2RewardTrainerParameters(
        learning_rate=0.005, multi_steps=6, action_names=["0", "1"]))
    tr = mgr.build_trainer({"state": _norm(2)}, use_gpu=True)
    assert tr.seq2reward_network.num_hiddens == 64 and tr.seq2reward_network.num_hidden_layers == 2
    for i in range(300):
        tr.train_batch(_game_batch(1024, i), i)
    b = _game_batch(64, 10_000)
    tr.validation_step(b, 0)
    s0 = torch.eye(2, device=DEV)
    q = get_Q(tr.seq2reward_network, s0, tr.all_permut).cpu()
    expected = torch.tensor([[6.0, 5.0], [5.0, 6.0]])
    assert float((q - expected).abs().max()) < 0.5, q
    torch.manual_seed(1)
    comp = mgr.compress_net_builder.build_value_network(_norm(2), output_dim=2).to(DEV)
    ct = CompressModelTrainer(comp, tr.seq2reward_network, mgr.trainer_param)
    for i in range(200):
        ct.train_batch(_game_batch(1024, 20_000 + i), i)
    _, _, _, acc = ct.validation_step(_game_batch(1024, 99_999), 0)
    assert acc >= 0.99, acc


def test_plan_at_the_sequence_limit():
    """A ** k = 65536 (A 2, k 16): the largest strides and workspace rows of the walk."""
    S, A, k, H, L, B = 2, 2, 16, 8, 1, 2
    net = _net(S, A, H, L)
    state = torch.randn(B, S, generator=torch.Generator().manual_seed(2)).to(DEV)
    q, q_all = net.plan(state, k, all_horizons=True)
    perm = gen_permutations(k, A).to(DEV)
    n = perm.shape[1]
    r = net(rlt.FeatureData(state.unsqueeze(0).repeat_interleave(n, dim=1)),
            rlt.FeatureData(perm.repeat(1, B, 1))).acc_reward
    assert torch.equal(q, r.reshape(B, A, n // A).max(dim=2).values)
    assert torch.equal(q, q_all[:, -1])
    assert _rel(q, O.get_q(_params64(net), state.cpu().double(), A, k, L)) < 1e-5


def test_plan_at_the_largest_tile():
    S, A, k, H, L, B = 252, 16, 2, 128, 4, 5
    net = _net(S, A, H, L)
    state = torch.randn(B, S, generator=torch.Generator().manual_seed(3)).to(DEV)
    _, q_all = net.plan(state, k, all_horizons=True)
    assert _rel(q_all, O.get_q_all(_params64(net), state.cpu().double(), A, k, L)) < 1e-5


def test_train_batch_without_valid_step_raises():
    params = Seq2RewardTrainerParameters(multi_steps=3, action_names=["0", "1"])
    tr = Seq2RewardTrainer(_net(2, 2, 8, 1), params).to(DEV)
    b = _batch(2, 2, 3, 8, 3)
    b.valid_step = None
    with pytest.raises(ValueError, match="valid_step"):
        tr.train_batch(b)


def _golden_updates(tr, arrays, meta, name):
    """Two reference-loop updates against the golden: yielded losses, the gradients of update 0,
    the weights after each update (Adam step budget) and the logged q_values."""
    rec = C.Recorder()
    tr.set_reporter(rec)
    for it in range(meta["n_updates"]):
        losses = run_update(tr, C.batch(arrays, it, DEV), it)
        want = arrays["losses"][it]
        for got, w in zip(losses, want):
            assert abs(float(got) - w) <= 1e-5 * max(1.0, abs(w)), (name, it, losses, want)
        if it == 0:
            for i, g in enumerate(tr.seq2reward_grads()):
                grad_close(sample(g), arrays[f"grad.{i}"], f"{name} grad.{i}")
            for i, g in enumerate(tr.step_predict_grads()):
                grad_close(sample(g), arrays[f"sgrad.{i}"], f"{name} sgrad.{i}")
        m = dict(meta, n_updates=it + 1)
        for i, p in enumerate(tr.seq2reward_network.parameters()):
            _adam_close(sample(p.detach()), torch.from_numpy(arrays[f"p{it + 1}.{i}"]), m)
        for i, p in enumerate(tr.step_predict_network.parameters()):
            _adam_close(sample(p.detach()), torch.from_numpy(arrays[f"sp{it + 1}.{i}"]), m)
    logged = [r["q_values"][0] for r in rec.logged if "q_values" in r]
    assert np.allclose(np.array(logged, dtype=np.float64).reshape(arrays["log.q_values"].shape),
                       arrays["log.q_values"], rtol=1e-4, atol=1e-5)


def _golden_validation(tr, arrays, name):
    mse, step, q_values, dist = tr.validation_step(C.batch(arrays, 0, DEV), 0)
    assert abs(mse - float(arrays["val.mse"])) <= 1e-4 * max(1.0, float(arrays["val.mse"])), name
    assert abs(step - float(arrays["val.step"])) <= 1e-4 * max(1.0, float(arrays["val.step"]))
    assert np.allclose(q_values, arrays["val.q_values"], rtol=1e-4, atol=1e-5)
    # an argmax may flip where two first actions are within the fp32 noise of each other
    B = arrays["batch0.reward"].shape[1]
    assert np.allclose(dist, arrays["val.action_distribution"], atol=1.5 / B)


@pytest.mark.parametrize("name", C.TRAINER_CASES)
def test_golden_trainer(name):
    arrays, meta = load(name)
    if name == "seq2reward_yaml":
        # seq2reward_test.yaml's trainer_param on the manager's default net builder
        from reagent_b200.model_managers import Seq2RewardModel
        mgr = Seq2RewardModel(trainer_param=C.trainer_params(meta))
        torch.manual_seed(meta["seed"])
        tr = mgr.build_trainer({"state": C.norm(meta["S"])}, use_gpu=True)
        C.check_digests(tr.seq2reward_network.parameters(), arrays, "p")
        C.check_digests(tr.step_predict_network.parameters(), arrays, "sp")
    else:
        tr = C.build_trainer(arrays, meta, DEV)
    b0 = C.batch(arrays, 0, DEV)
    out = tr.seq2reward_network(b0.state, b0.action, b0.valid_step.flatten()).acc_reward
    n = arrays["out.acc_reward"].shape[0]
    assert rel_err(out[:n], arrays["out.acc_reward"]) < 1e-5
    assert rel_err(tr.get_mse_loss(b0), arrays["loss.mse"]) < 1e-5
    assert rel_err(tr.get_step_entropy_loss(b0), arrays["loss.step"]) < 1e-5
    _golden_updates(tr, arrays, meta, name)
    _golden_validation(tr, arrays, name)


@pytest.mark.parametrize("name", C.COMPRESS_CASES)
def test_golden_compress(name):
    arrays, meta = load(name)
    tr, net = C.build_compress(arrays, meta, DEV)
    b0 = C.batch(arrays, 0, DEV)
    q = get_Q(net, b0.state.float_features[0], tr.all_permut)
    assert rel_err(q, arrays["q"]) < 1e-5
    mse, acc = tr.get_loss(b0)
    assert rel_err(mse, arrays["loss.mse"]) < 1e-5
    assert float(acc) == float(arrays["loss.accuracy"])
    rec = C.Recorder()
    tr.set_reporter(rec)
    for it in range(meta["n_updates"]):
        (loss,) = run_update(tr, C.batch(arrays, it, DEV), it)
        w = arrays["losses"][it]
        assert abs(float(loss) - w) <= 1e-5 * max(1.0, abs(w))
        if it == 0:
            for i, g in enumerate(tr.compress_grads()):
                grad_close(sample(g), arrays[f"cgrad.{i}"], f"{name} cgrad.{i}")
        m = dict(meta, n_updates=it + 1)
        for i, p in enumerate(tr.compress_model_network.parameters()):
            _adam_close(sample(p.detach()), torch.from_numpy(arrays[f"cp{it + 1}.{i}"]), m)
    # after an update an argmax may flip where two outputs are within the fp32 noise
    B = arrays["batch0.reward"].shape[1]
    assert np.allclose([r["accuracy"] for r in rec.logged], arrays["log.accuracy"], atol=1.5 / B)
    mse, q_values, dist, acc = tr.validation_step(b0, 0)
    assert abs(mse - float(arrays["val.mse"])) <= 1e-4 * max(1.0, float(arrays["val.mse"]))
    assert np.allclose(q_values, arrays["val.q_values"], rtol=1e-4, atol=1e-5)
    assert np.allclose(dist, arrays["val.action_distribution"], atol=1.5 / B)
    assert abs(acc - float(arrays["val.accuracy"])) <= 1.5 / B


@pytest.mark.parametrize("name", C.PLAN_CASES)
def test_golden_plan(name):
    arrays, meta = load(name)
    net = C.plan_network(arrays, meta, DEV)
    state = torch.from_numpy(arrays["state"]).to(DEV)
    q, q_all = net.plan(state, meta["k"], all_horizons=True)
    assert rel_err(q_all, arrays["q_all"]) < 1e-5
    assert rel_err(q, arrays["q"]) < 1e-5
    assert torch.equal(get_Q(net, state, torch.from_numpy(arrays["permutations"])), q)
