"""ParametricDQN end to end on the GPU: the fused tiled next-action forward
(rb200_mlp_forward_tiled) against the materialised repeat + cat + rb200_mlp_forward it replaces,
bit for bit; ParametricDQNTrainer.train_batch against that materialised path; the replay batch
sample_parametric_dqn_batch, the ParametricDQN manager at both CartPole configurations and its
policy against golden vectors of the unmodified reference (oracle/make_parametric_golden.py:
ParametricDqnInputMaker, the reference trainer, parametric_dqn_scorer + SoftmaxActionSampler);
the captured online step (FusedDqnStep) against the eager updates it captures."""
import random

import numpy as np
import pytest
import torch

from tests import golden_util as G
from tests.online_step import drawn_indices, online_steps
from tests.golden_cases import CARTPOLE_CASES, INPUTMAKER_CASES, PDQN_CASES, cartpole_batch

pytestmark = pytest.mark.gpu

E_INVALID, E_SMEM = -1, -3


def _bits(t):
    return t.contiguous().view(torch.int32)


def _bit_equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _critic(S, K, sizes, acts, out_dim=1, seed=0):
    from reagent_b200.models import FullyConnectedCritic

    torch.manual_seed(seed)
    return FullyConnectedCritic(S, K, sizes, acts, output_dim=out_dim).cuda()


def _materialised(arena, state, actions, M):
    from reagent_b200.models.arena import run_mlp

    x = torch.cat((state.repeat_interleave(M, dim=0), actions), dim=1).contiguous()
    out = torch.empty(x.shape[0], arena.dims[-1], device=x.device)
    run_mlp(arena.desc(), x, out)
    return out


def _tiled(arenas, state, actions, M):
    from reagent_b200.models.arena import run_mlp_tiled

    outs = [torch.empty(actions.shape[0], a.dims[-1], device=actions.device) for a in arenas]
    run_mlp_tiled(arenas, state, actions, M, outs)
    return outs


def _check_tiled(S, K, M, B, sizes, acts, out_dim=1, one_hot=False, n_nets=2, seed=0):
    q = _critic(S, K, sizes, acts, out_dim, seed)
    qt = q.get_target_network()
    with torch.no_grad():  # a target that differs from the online network
        for p in qt.parameters():
            p.add_(0.01 * torch.randn_like(p))
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    state = torch.randn(B, S, device="cuda", generator=g)
    if one_hot:
        assert K == M
        actions = torch.eye(M, device="cuda").repeat(B, 1)
    else:
        actions = torch.randn(B * M, K, device="cuda", generator=g)
    arenas = [qt.arena, q.arena][:n_nets]
    got = _tiled(arenas, state, actions, M)
    torch.cuda.synchronize()
    for a, o in zip(arenas, got):
        want = _materialised(a, state, actions, M)
        assert torch.isfinite(want).all()
        assert _bit_equal(o, want), (S, K, M, B, sizes, acts)
    if n_nets == 2:  # the two networks really differ, so each output is its own network's
        assert not torch.equal(got[0], got[1])


# ---------------------------------------------------------------------------
# rb200_mlp_forward_tiled against the materialised input
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 2, 3, 16, 33, 128])
def test_tiled_forward_one_hot_actions(M):
    _check_tiled(S=128, K=M, M=M, B=37, sizes=[256, 128], acts=["relu", "relu"], one_hot=True)


@pytest.mark.parametrize("K,M", [(5, 7), (9, 2), (40, 3)])
def test_tiled_forward_feature_actions(K, M):
    _check_tiled(S=24, K=K, M=M, B=29, sizes=[64, 32], acts=["relu", "relu"])


# rows = B*M on both sides of the 16/32-row tile switch (16 * 132 SMs = 2112 rows) and ragged
@pytest.mark.parametrize("B,M", [(1, 1), (5, 3), (704, 3), (2112, 1), (2113, 1), (705, 3),
                                 (4096, 2), (331, 16)])
def test_tiled_forward_row_counts(B, M):
    _check_tiled(S=17, K=6, M=M, B=B, sizes=[48, 40], acts=["relu", "tanh"])


@pytest.mark.parametrize("S,K", [(4, 2), (5, 2), (3, 3), (126, 3), (1, 1)])
def test_tiled_forward_widths_not_multiple_of_4(S, K):
    _check_tiled(S=S, K=K, M=K, B=301, sizes=[33, 17], acts=["leaky_relu", "leaky_relu"],
                 one_hot=True)


def test_tiled_forward_one_layer_network():
    _check_tiled(S=13, K=4, M=4, B=257, sizes=[], acts=[], one_hot=True)


@pytest.mark.parametrize("act", ["relu", "tanh", "leaky_relu"])
def test_tiled_forward_activations(act):
    _check_tiled(S=32, K=8, M=8, B=300, sizes=[64, 64, 32], acts=[act] * 3, out_dim=3,
                 one_hot=True)


# rows > 2112 (32-row tiles allowed) with S+K = 132: the hidden width alone decides the tile.
# shared floats = 2*stage(KC) + R*(ld_in + 2*ld_h + ld_o) <= 227 KB picks, in order,
#   512 threads / KC 32 (hidden 512), 512 / 16 (640), 256 / 32 (1024), 256 / 16 (1280)
@pytest.mark.parametrize("hidden", [512, 640, 1024, 1280])
def test_tiled_forward_every_row_tile(hidden):
    _check_tiled(S=116, K=16, M=16, B=160, sizes=[hidden], acts=["relu"], one_hot=True)


@pytest.mark.parametrize("cfg", ["512,32", "512,16", "256,32", "256,16"])
def test_tiled_forward_forced_tiles(cfg, monkeypatch):
    # RB200_FORCE_CFG is read by the tile choice of both entry points alike
    monkeypatch.setenv("RB200_FORCE_CFG", cfg)
    _check_tiled(S=20, K=5, M=5, B=97, sizes=[96, 48], acts=["relu", "relu"], one_hot=True)


@pytest.mark.parametrize("n_nets", [1, 2])
def test_tiled_forward_one_or_two_networks(n_nets):
    _check_tiled(S=30, K=6, M=6, B=513, sizes=[128, 64], acts=["relu", "relu"], out_dim=2,
                 one_hot=True, n_nets=n_nets)


def test_tiled_forward_rejects_bad_arguments():
    from reagent_b200 import _lib

    lib = _lib.lib()
    q = _critic(6, 3, [16], ["relu"])
    other = _critic(6, 3, [24], ["relu"])
    state = torch.zeros(4, 6, device="cuda")
    act = torch.zeros(12, 3, device="cuda")
    o0, o1 = torch.zeros(12, 1, device="cuda"), torch.zeros(12, 1, device="cuda")
    s = _lib.cur_stream()

    def call(n0=q.arena.desc(), n1=None, st=state.data_ptr(), S=6, a=act.data_ptr(), K=3, B=4,
             M=3, out0=o0.data_ptr(), out1=None):
        return lib.rb200_mlp_forward_tiled(n0, n1, st, S, a, K, B, M, out0, out1, s)

    assert call() == 0
    assert call(n1=q.get_target_network().arena.desc(), out1=o1.data_ptr()) == 0
    assert call(st=None) == E_INVALID
    assert call(a=None) == E_INVALID
    assert call(out0=None) == E_INVALID
    assert call(n0=None) == E_INVALID
    assert call(n1=q.arena.desc()) == E_INVALID          # net1 without out1
    assert call(out1=o1.data_ptr()) == E_INVALID          # out1 without net1
    assert call(n1=other.arena.desc(), out1=o1.data_ptr()) == E_INVALID  # differing dims
    assert call(S=5) == E_INVALID                          # widths != dims[0]
    assert call(K=4) == E_INVALID
    assert call(S=0, K=9) == E_INVALID
    assert call(B=0) == E_INVALID
    assert call(M=0) == E_INVALID
    assert call(B=1 << 16, M=1 << 15) == E_INVALID         # B*M past int32
    assert "int32" in lib.rb200_last_error().decode()
    wide = _critic(6, 3, [16], ["relu"], out_dim=1100)    # output tile too wide
    assert call(n0=wide.arena.desc()) == E_SMEM
    huge = _critic(6, 3, [6000], ["relu"])                # hidden tile past 227 KB
    assert call(n0=huge.arena.desc()) == E_SMEM
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# ParametricDQNTrainer: the fused path against the materialised one
# ---------------------------------------------------------------------------
def _materialise_trainer_forward(monkeypatch):
    """Make the trainer score the tiled next actions the way it did before the fused kernel:
    repeat + cat in torch, then one rb200_mlp_forward per network."""
    import reagent_b200.training.parametric_dqn_trainer as mod

    def run(arenas, state, actions, M, outs):
        for a, o in zip(arenas, outs):
            o.copy_(_materialised(a, state, actions, M))

    monkeypatch.setattr(mod, "run_mlp_tiled", run)


def _pdqn_from_golden(name):
    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import ParametricDQNTrainer

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
    return t, batch, meta["n_updates"]


def _trainer_state(t):
    nets = [t.q_network, t.q_network_target]
    if t.reward_network is not None:
        nets.append(t.reward_network)
    return [p.detach().clone() for n in nets for p in n.parameters()]


def _run_updates(t, batch, n):
    out = []
    for it in range(n):
        loss = t.train_batch(batch, it).clone()
        out.append((loss, t._ws["td_target"].clone(),
                    None if t.reward_network is None else t._ws["r_loss"].clone()))
    torch.cuda.synchronize()
    return out


def _assert_same_run(run0, run1, state0, state1):
    for (l0, td0, r0), (l1, td1, r1) in zip(run0, run1):
        assert _bit_equal(l0, l1) and _bit_equal(td0, td1)
        assert (r0 is None) == (r1 is None) and (r0 is None or _bit_equal(r0, r1))
    assert len(state0) == len(state1)
    assert all(_bit_equal(a, b) for a, b in zip(state0, state1))


@pytest.mark.parametrize("name", PDQN_CASES)
def test_trainer_golden_cases_bit_equal_to_materialised(name, monkeypatch):
    t, batch, n = _pdqn_from_golden(name)
    fused = _run_updates(t, batch, n)
    fused_state = _trainer_state(t)
    _materialise_trainer_forward(monkeypatch)
    t2, batch2, _ = _pdqn_from_golden(name)
    ref = _run_updates(t2, batch2, n)
    _assert_same_run(fused, ref, fused_state, _trainer_state(t2))


def _big_trainer(seed):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import ParametricDQNTrainer

    S, A = 128, 16
    q = _critic(S, A, [256, 128], ["relu", "relu"], seed=seed)
    rn = _critic(S, A, [256, 128], ["relu", "relu"], seed=seed + 1)
    return ParametricDQNTrainer(q, q.get_target_network(), rn,
                                rl=RLParameters(gamma=0.99, target_update_rate=0.1),
                                double_q_learning=True,
                                optimizer=Optimizer__Union(AdamW={"lr": 1e-3, "amsgrad": True})).cuda()


def _big_batch(S=128, A=16, B=4096):
    from reagent_b200.core import types as rlt

    g = torch.Generator(device="cuda").manual_seed(11)
    a = torch.randint(A, (B,), device="cuda", generator=g)
    na = torch.randint(A, (B,), device="cuda", generator=g)
    nt = (torch.rand(B, 1, device="cuda", generator=g) > 0.05).float()
    eye = torch.eye(A, device="cuda").repeat(B, 1)
    return rlt.ParametricDqnInput(
        state=rlt.FeatureData(torch.randn(B, S, device="cuda", generator=g)),
        next_state=rlt.FeatureData(torch.randn(B, S, device="cuda", generator=g)),
        reward=torch.randn(B, 1, device="cuda", generator=g), time_diff=None, step=None,
        not_terminal=nt, action=rlt.FeatureData(torch.nn.functional.one_hot(a, A).float()),
        next_action=rlt.FeatureData(torch.nn.functional.one_hot(na, A).float() * nt),
        possible_actions=rlt.FeatureData(eye), possible_actions_mask=torch.ones(B, A, device="cuda"),
        possible_next_actions=rlt.FeatureData(eye),
        possible_next_actions_mask=torch.ones(B, A, device="cuda"), extras=rlt.ExtraData())


def test_trainer_large_batch_bit_equal_to_materialised(monkeypatch):
    t, batch = _big_trainer(3), _big_batch()
    fused = _run_updates(t, batch, 2)
    fused_state = _trainer_state(t)
    _materialise_trainer_forward(monkeypatch)
    t2 = _big_trainer(3)
    ref = _run_updates(t2, batch, 2)
    _assert_same_run(fused, ref, fused_state, _trainer_state(t2))


# ---------------------------------------------------------------------------
# sample_parametric_dqn_batch against ParametricDqnInputMaker on sample_transition_batch
# ---------------------------------------------------------------------------
def _transitions(n, S, A, seed, log_prob=False, priority=False, p_term=0.05):
    rng = np.random.RandomState(seed)
    d = dict(observation=rng.randn(n, S).astype(np.float32),
             action=rng.randint(0, A, n).astype(np.int64),
             reward=rng.randn(n).astype(np.float32), terminal=rng.rand(n) < p_term)
    if log_prob:
        d["log_prob"] = np.log(rng.uniform(0.05, 1.0, n)).astype(np.float32)
    if priority:
        d["priority"] = rng.uniform(0.1, 10.0, n)
    return d


def _input_maker(tb, A):
    """ParametricDqnInputMaker.__call__ (trainer_preprocessor.py:376-413) on a transition batch."""
    import torch.nn.functional as F

    B = tb.state.shape[0]
    term = tb.terminal
    action = F.one_hot(tb.action.reshape(-1), A).float()
    next_action = torch.zeros_like(action)
    keep = (term == 0).reshape(-1)
    next_action[keep] = F.one_hot(tb.next_action.reshape(-1)[keep], A).float()
    pa = torch.eye(A, device=action.device).repeat(B, 1)
    return dict(state=tb.state, next_state=tb.next_state, action=action,
                next_action=next_action, reward=tb.reward, not_terminal=1.0 - term.float(),
                possible_actions=pa, possible_next_actions=pa.clone(),
                possible_actions_mask=torch.ones(B, A, device=action.device),
                possible_next_actions_mask=torch.ones(B, A, device=action.device))


@pytest.mark.parametrize("case", ["h1_terminal", "h3_wrap", "log_prob", "prioritized"])
def test_sampler_matches_input_maker(case):
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, ReplayBuffer

    S, A, B, cap = 7, 3, 300, 512
    horizon = 3 if case == "h3_wrap" else 1
    prioritized = case == "prioritized"
    # h3_wrap writes past the capacity, so the cursor wraps and n-step windows cross the end
    n = 700 if case == "h3_wrap" else 450
    data = _transitions(n, S, A, 5, log_prob=case == "log_prob", priority=prioritized,
                        p_term=0.2 if case == "h1_terminal" else 0.05)
    cls = PrioritizedReplayBuffer if prioritized else ReplayBuffer
    rb = cls(stack_size=1, replay_capacity=cap, batch_size=B, update_horizon=horizon, gamma=0.9)
    rb.add_batch(**data)
    valid = rb._is_index_valid.nonzero().reshape(-1)
    idx = valid[torch.randint(len(valid), (B,), generator=torch.Generator().manual_seed(2))]
    got = rb.sample_parametric_dqn_batch(B, A, indices=idx)
    tb = rb.sample_transition_batch(B, indices=idx)
    want = _input_maker(tb, A)
    assert got.step is None and got.time_diff is None
    assert torch.equal(got.indices.reshape(-1).cpu(), idx)
    for k in ("state", "next_state", "action", "next_action", "possible_actions",
              "possible_next_actions"):
        assert _bit_equal(getattr(got, k).float_features, want[k]), k
    for k in ("reward", "not_terminal", "possible_actions_mask", "possible_next_actions_mask"):
        assert _bit_equal(getattr(got, k), want[k].reshape(getattr(got, k).shape)), k
    if case == "h1_terminal":
        assert (got.not_terminal == 0).any()
    if case == "log_prob":
        assert _bit_equal(got.extras.action_probability, tb.log_prob.exp())
    else:
        assert got.extras.action_probability is None
    disc = rb.sample_discrete_dqn_batch(B, A, indices=idx)
    if prioritized:
        assert _bit_equal(got.sampling_probabilities, disc.sampling_probabilities)
    else:
        assert got.sampling_probabilities is None


def test_sampler_ignores_a_stored_mask_and_draws_like_the_discrete_batch():
    from reagent_b200.replay_memory import ReplayBuffer

    S, A, B = 5, 4, 64
    data = _transitions(300, S, A, 9)
    data["possible_actions_mask"] = np.zeros((300, A), dtype=np.float32)
    rb = ReplayBuffer(stack_size=1, replay_capacity=512, batch_size=B)
    rb.add_batch(**data)
    torch.manual_seed(4)
    got = rb.sample_parametric_dqn_batch(B, A)
    torch.manual_seed(4)
    disc = rb.sample_discrete_dqn_batch(B, A)
    assert torch.equal(got.indices, disc.indices)
    assert torch.equal(got.action.float_features, disc.action)
    assert torch.equal(got.possible_actions_mask, torch.ones(B, A, device="cuda"))
    assert torch.equal(disc.possible_actions_mask, torch.zeros(B, A, device="cuda"))


# ---------------------------------------------------------------------------
# the ParametricDQN manager and its policy
# ---------------------------------------------------------------------------
def _norm(S, A):
    from reagent_b200.core.parameters import NormalizationData, NormalizationParameters as NP

    return {"state": NormalizationData({i: NP("CONTINUOUS", mean=0.0, stddev=1.0) for i in range(S)}),
            "action": NormalizationData({100 + i: NP("DISCRETE_ACTION") for i in range(A)})}


def _cartpole_manager(sarsa):
    """gym/tests/configs/cartpole/parametric_{dqn,sarsa}_cartpole_online.yaml as written."""
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.model_managers import ParametricDQN
    from reagent_b200.net_builder import ParametricFullyConnected
    from reagent_b200.optimizer import Optimizer__Union

    if sarsa:
        return ParametricDQN(
            rl=RLParameters(gamma=0.99, target_update_rate=0.2, maxq_learning=False, temperature=0.35),
            double_q_learning=True, minibatches_per_step=1,
            optimizer=Optimizer__Union(Adam={"lr": 0.05}),
            net_builder=ParametricFullyConnected(sizes=[64, 64], activations=["leaky_relu"] * 2),
            eval_parameters=EvaluationParameters(calc_cpe_in_training=False))
    return ParametricDQN(
        rl=RLParameters(gamma=0.99, target_update_rate=0.1, maxq_learning=True, temperature=1.0),
        double_q_learning=True, minibatches_per_step=1,
        optimizer=Optimizer__Union(AdamW={"lr": 0.001, "amsgrad": True}),
        net_builder=ParametricFullyConnected(sizes=[128, 64], activations=["leaky_relu"] * 2),
        eval_parameters=EvaluationParameters(calc_cpe_in_training=False))


@pytest.mark.parametrize("sarsa", [False, True])
def test_manager_builds_and_trains_the_cartpole_configs(sarsa, monkeypatch):
    from reagent_b200.core import types as rlt
    from reagent_b200.optimizer import FusedAdam, FusedAdamW, SoftUpdate
    from reagent_b200.replay_memory import ReplayBuffer
    from reagent_b200.training import ParametricDQNTrainer

    m = _cartpole_manager(sarsa)
    torch.manual_seed(0)
    t = m.build_trainer(_norm(4, 2), use_gpu=True)
    assert type(t) is ParametricDQNTrainer and t.num_actions == 2
    sizes = [64, 64] if sarsa else [128, 64]
    assert t.q_network.arena.dims == [6] + sizes + [1]
    assert t.reward_network.arena.dims == [6] + sizes + [1]
    assert t.maxq_learning == (not sarsa) and t.double_q_learning
    opts = t.optimizers()
    assert [type(o) for o in opts] == [FusedAdam if sarsa else FusedAdamW] * 2 + [SoftUpdate]
    for a, b in zip(t.q_network.parameters(), t.q_network_target.parameters()):
        assert torch.equal(a, b) and a.data_ptr() != b.data_ptr()
    # metrics to score widen the reward network
    class RO:
        metric_reward_values = {"b": 1.0, "a": 2.0}
    t2 = m.build_trainer(_norm(4, 2), use_gpu=True, reward_options=RO())
    assert t2.reward_network.arena.dims[-1] == 3
    with pytest.raises(RuntimeError):
        m.build_trainer(_norm(4, 2), use_gpu=False)

    # trains from replay batches; the update equals the materialised path bit for bit
    rb = ReplayBuffer(stack_size=1, replay_capacity=4096, batch_size=1024)
    rb.add_batch(**_transitions(3000, 4, 2, 1))
    torch.manual_seed(5)
    batches = [rb.sample_parametric_dqn_batch(1024, 2) for _ in range(5)]
    assert isinstance(batches[0], rlt.ParametricDqnInput)
    losses = [t.train_batch(b).clone() for b in batches]
    state = _trainer_state(t)
    _materialise_trainer_forward(monkeypatch)
    torch.manual_seed(0)
    t3 = m.build_trainer(_norm(4, 2), use_gpu=True)
    ref = [t3.train_batch(b).clone() for b in batches]
    torch.cuda.synchronize()
    assert all(torch.isfinite(l).all() for l in losses)
    assert all(_bit_equal(a, b) for a, b in zip(losses, ref))
    assert all(_bit_equal(a, b) for a, b in zip(state, _trainer_state(t3)))


@pytest.mark.parametrize("sarsa", [False, True])
def test_policy_scores_and_softmax_draws(sarsa):
    from reagent_b200.core import types as rlt
    from reagent_b200.gym.policies import SoftmaxActionSampler

    m = _cartpole_manager(sarsa)
    torch.manual_seed(0)
    t = m.build_trainer(_norm(4, 2), use_gpu=True)
    policy = m.create_policy(t)
    with pytest.raises(NotImplementedError):
        m.create_policy(t, serving=True)
    assert isinstance(policy.sampler, SoftmaxActionSampler)
    assert policy.sampler.temperature == (0.35 if sarsa else 1.0)
    obs = torch.randn(9, 4, generator=torch.Generator().manual_seed(3))
    scores = policy.scorer(rlt.FeatureData(obs))
    assert scores.shape == (9, 2) and t.q_network.training
    # the reference scorer: q_network(tiled_state, identity tiling).view(-1, A)
    tiled = rlt.FeatureData(obs.cuda().repeat_interleave(2, dim=0))
    eye = rlt.FeatureData(torch.eye(2, device="cuda").repeat(9, 1))
    want = t.q_network(tiled, eye).view(-1, 2)
    assert _bit_equal(scores, want)
    torch.manual_seed(42)
    act = policy.act(rlt.FeatureData(obs))
    torch.manual_seed(42)
    idx = torch.distributions.Categorical(logits=want / policy.sampler.temperature).sample()
    assert torch.equal(act.action.argmax(1), idx.cpu())
    assert act.action.device.type == "cpu"


# ---------------------------------------------------------------------------
# the captured online step
# ---------------------------------------------------------------------------
S_ON, A_ON, B_ON, CAP_ON = 12, 3, 256, 4096


def _online_trainer():
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import ParametricDQNTrainer

    q = _critic(S_ON, A_ON, [48, 32], ["leaky_relu", "leaky_relu"], seed=1)
    rn = _critic(S_ON, A_ON, [48, 32], ["leaky_relu", "leaky_relu"], seed=2)
    return ParametricDQNTrainer(q, q.get_target_network(), rn,
                                rl=RLParameters(gamma=0.9, target_update_rate=0.05),
                                double_q_learning=True,
                                optimizer=Optimizer__Union(AdamW={"lr": 1e-3, "amsgrad": True})).cuda()


def _online_setup(prioritized, seed=3):
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, ReplayBuffer

    cls = PrioritizedReplayBuffer if prioritized else ReplayBuffer
    rb = cls(stack_size=1, replay_capacity=CAP_ON, batch_size=B_ON)
    rb.add_batch(**_transitions(3000, S_ON, A_ON, seed, priority=prioritized))
    return rb, _online_trainer()


@pytest.mark.parametrize("prefetch", [False, True])
def test_online_host_step_equals_eager(prefetch):
    from reagent_b200.training.fused_step import FusedDqnStep

    n = 30
    rb, t = _online_setup(False)
    torch.manual_seed(7)
    eager = []
    for _ in range(n + 1):  # the constructor's warm-up is update 0
        # the step draws torch.randint ranks on the host, as the eager sample does
        eager.append(float(t.train_batch(rb.sample_parametric_dqn_batch(B_ON, A_ON))))
    rb2, t2 = _online_setup(False)
    torch.manual_seed(7)
    fused = FusedDqnStep(t2, rb2, B_ON, prefetch=prefetch)
    got = []
    for _ in range(n):
        lh = fused.step()
        torch.cuda.synchronize()
        got.append(float(lh[0]))
    assert got == eager[1:]
    assert all(_bit_equal(a, b) for a, b in zip(_trainer_state(t), _trainer_state(t2)))


def test_online_device_step_equals_eager_and_host_replica():
    from reagent_b200.training.fused_step import FusedDqnStep

    extra = _transitions(30, S_ON, A_ON, 8, priority=True)
    runs = []
    for captured in (True, False):
        rb, t = _online_setup(True, seed=7)
        random.seed(5)
        fused = FusedDqnStep(t, rb, B_ON, rng="device", online=True)
        losses, idx = [], []
        for loss in online_steps(fused, extra, 30, captured):
            losses.append(loss)
            idx.append(drawn_indices(fused))
        runs.append((losses, idx, _trainer_state(t)))
    (l0, i0, p0), (l1, i1, p1) = runs
    assert l0 == l1 and all(np.isfinite(l0))
    assert all(np.array_equal(a, b) for a, b in zip(i0, i1))
    assert all(_bit_equal(a, b) for a, b in zip(p0, p1))

    # the device draws are the host buffer's draws with Python's random stream
    rb_h, _ = _online_setup(True, seed=7)
    random.seed(5)
    host = [rb_h.sample_parametric_dqn_batch(B_ON, A_ON).indices.cpu().numpy().reshape(-1)]
    for i in range(30):
        rb_h.add(**{k: (v[i].item() if np.ndim(v[i]) == 0 else v[i]) for k, v in extra.items()})
        host.append(rb_h.sample_parametric_dqn_batch(B_ON, A_ON).indices.cpu().numpy().reshape(-1))
    assert all(np.array_equal(a, b) for a, b in zip(host[1:], i0))


def test_online_step_refuses_per_and_shards():
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    rb, t = _online_setup(True)
    with pytest.raises(NotImplementedError):
        FusedDqnStep(t, rb, B_ON, rng="device", online=True, per=PrioritizedUpdate())
    with pytest.raises(NotImplementedError):
        FusedDqnStep(t, rb, B_ON, shard=(0, 2))
    with pytest.raises(NotImplementedError):
        FusedDqnStep(t, rb, B_ON, process_group=object())


# ---------------------------------------------------------------------------
# against the reference's goldens (oracle/make_parametric_golden.py)
# ---------------------------------------------------------------------------


def _golden_buffer(arrays, meta, bulk):
    from reagent_b200.replay_memory import PrioritizedReplayBuffer, ReplayBuffer

    cls = PrioritizedReplayBuffer if meta["prioritized"] else ReplayBuffer
    rb = cls(stack_size=1, replay_capacity=meta["cap"], batch_size=meta["B"],
             update_horizon=meta["horizon"], gamma=meta["gamma"])
    st = {k: arrays[f"stream.{k}"] for k in meta["keys"]}
    if bulk:
        rb.add_batch(**st)
        return rb
    for t in range(meta["n_add"]):
        kw = {}
        for k, v in st.items():
            v = v[t]
            if k == "terminal":
                v = bool(v)
            elif k == "priority":
                v = float(v)
            elif k == "action":
                v = int(v)
            elif np.ndim(v) == 0:
                v = float(v)
            kw[k] = v
        rb.add(**kw)
    return rb


def _eq(name, got, want, keep=None):
    got = got.detach().cpu().numpy()
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape)
    if keep is not None:
        got, want = got[keep], want[keep]
    assert np.array_equal(got, want), name


@pytest.mark.parametrize("bulk", [False, True])
@pytest.mark.parametrize("name", INPUTMAKER_CASES)
def test_sampler_matches_reference_inputmaker(name, bulk):
    """sample_parametric_dqn_batch at the reference's drawn indices against the reference's
    sample_transition_batch + ParametricDqnInputMaker, field by field."""
    arrays, meta = G.load(name)
    rb = _golden_buffer(arrays, meta, bulk)
    B, A = meta["B"], meta["A"]
    for s_i in range(meta["n_samples"]):
        pre = f"sample{s_i}."
        idx = torch.from_numpy(arrays[pre + "indices"].reshape(-1).copy())
        out = rb.sample_parametric_dqn_batch(B, A, indices=idx)
        assert out.step is None and out.time_diff is None
        _eq(pre + "indices", out.indices, arrays[pre + "indices"])
        # the reference leaves next_state undefined on terminal rows
        # (circular_replay_buffer.py:621): compared on non-terminal rows only
        nonterm = ~arrays[pre + "terminal"].reshape(-1)
        _eq(pre + "state", out.state.float_features, arrays[pre + "state"])
        _eq(pre + "next_state", out.next_state.float_features, arrays[pre + "next_state"], nonterm)
        _eq(pre + "not_terminal", out.not_terminal, arrays[pre + "not_terminal"])
        _eq(pre + "action", out.action.float_features, arrays[pre + "action"])
        _eq(pre + "next_action", out.next_action.float_features, arrays[pre + "next_action"])
        for k in ("possible_actions", "possible_next_actions"):
            _eq(pre + k, getattr(out, k).float_features, arrays[pre + k])
        for k in ("possible_actions_mask", "possible_next_actions_mask"):
            _eq(pre + k, getattr(out, k), arrays[pre + k])
        if meta["horizon"] == 1:
            _eq(pre + "reward", out.reward, arrays[pre + "reward"])
        else:  # n-step fold: the same fp32 products, summed in an order torch may not share
            np.testing.assert_allclose(out.reward.cpu().numpy(), arrays[pre + "reward"],
                                       rtol=2e-6, atol=1e-6)
        # exp() on the device against the host: 1 ulp
        np.testing.assert_allclose(out.extras.action_probability.cpu().numpy(),
                                   arrays[pre + "action_probability"], rtol=3e-7, atol=0)


def _golden_manager(meta):
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.model_managers import ParametricDQN
    from reagent_b200.net_builder import ParametricFullyConnected
    from reagent_b200.optimizer import Optimizer__Union

    kw = {"lr": meta["lr"]}
    if meta["optimizer"] == "AdamW":
        kw.update(amsgrad=meta["amsgrad"], weight_decay=meta["weight_decay"])
    return ParametricDQN(
        rl=RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"],
                        maxq_learning=meta["maxq"], temperature=meta["temperature"]),
        double_q_learning=meta["double_q"], minibatches_per_step=1,
        optimizer=Optimizer__Union(**{meta["optimizer"]: kw}),
        net_builder=ParametricFullyConnected(sizes=meta["sizes"], activations=meta["acts"]),
        eval_parameters=EvaluationParameters(calc_cpe_in_training=False))


@pytest.mark.parametrize("name", CARTPOLE_CASES)
def test_manager_trains_like_the_reference_cartpole(name):
    """ParametricDQN(...).build_trainer at the CartPole configuration, started from the
    reference's weights and trained on its five batches: losses and all three networks to 1e-5."""
    from reagent_b200.core import types as rlt

    arrays, meta = G.load(name)
    t = _golden_manager(meta).build_trainer(_norm(meta["S"], meta["A"]), use_gpu=True)
    G.load_into_module(arrays, "q0", t.q_network)
    G.load_into_module(arrays, "qt0", t.q_network_target)
    G.load_into_module(arrays, "r0", t.reward_network)
    for it in range(meta["n_updates"]):
        b = cartpole_batch(arrays, it, "cuda")
        batch = rlt.ParametricDqnInput(
            state=rlt.FeatureData(b["state"]), next_state=rlt.FeatureData(b["next_state"]),
            reward=b["reward"], time_diff=None, step=None, not_terminal=b["not_terminal"],
            action=rlt.FeatureData(b["action"]), next_action=rlt.FeatureData(b["next_action"]),
            possible_actions=rlt.FeatureData(b["possible_actions"]),
            possible_actions_mask=b["possible_actions_mask"],
            possible_next_actions=rlt.FeatureData(b["possible_next_actions"]),
            possible_next_actions_mask=b["possible_next_actions_mask"], extras=rlt.ExtraData())
        td = float(t.train_batch(batch, it))
        rl_ = float(t._ws["r_loss"])
        for got, want in ((td, arrays["losses"][it][0]), (rl_, arrays["losses"][it][1])):
            assert abs(got - want) <= 1e-5 * max(1.0, abs(want)), (it, got, want)
    for net, prefix in ((t.q_network, "qN"), (t.q_network_target, "qtN"), (t.reward_network, "rN")):
        ps = list(net.parameters())
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-5 and G.rel_err(ps[2 * i + 1], b) < 1e-5, (prefix, i)


@pytest.mark.parametrize("ti", [0, 1])
def test_policy_matches_reference_scorer_and_draws(ti):
    """create_policy's scorer against the reference's parametric_dqn_scorer to 1e-5, and the
    seeded SoftmaxActionSampler draws on those scores equal to the reference's."""
    from reagent_b200.core import types as rlt

    arrays, meta = G.load("parametric_scorer")
    temp = meta["temperatures"][ti]
    m = _golden_manager(dict(lr=1e-3, optimizer="Adam", gamma=0.99, tau=0.1, maxq=True,
                             temperature=temp, double_q=True, sizes=meta["sizes"],
                             acts=meta["acts"]))
    t = m.build_trainer(_norm(meta["S"], meta["A"]), use_gpu=True)
    G.load_into_module(arrays, "q", t.q_network)
    policy = m.create_policy(t)
    assert policy.sampler.temperature == temp
    scores = policy.scorer(rlt.FeatureData(torch.from_numpy(arrays["obs"])))
    assert t.q_network.training
    assert scores.shape == tuple(arrays["scores"].shape)
    assert G.rel_err(scores, arrays["scores"]) < 1e-5
    # torch's CUDA and CPU generators are different streams: the reference's draws are CPU draws
    cpu_scores = scores.cpu()
    for d in range(meta["n_draws"]):
        torch.manual_seed(meta["seed"] + 100 * (ti + 1) + d)
        out = policy.sampler.sample_action(cpu_scores)
        assert torch.equal(out.action, torch.from_numpy(arrays[f"t{ti}.d{d}.action"]))
        np.testing.assert_allclose(out.log_prob.numpy(), arrays[f"t{ti}.d{d}.log_prob"],
                                   rtol=1e-5, atol=1e-6)


def test_tiled_wrapper_checks_tensor_shapes():
    """run_mlp_tiled checks what the C ABI cannot see: row counts, widths, dtype, layout."""
    from reagent_b200.models.arena import run_mlp_tiled

    q = _critic(6, 3, [16], ["relu"])
    a = [q.arena]
    st, act, out = (torch.zeros(4, 6, device="cuda"), torch.zeros(12, 3, device="cuda"),
                    torch.zeros(12, 1, device="cuda"))
    run_mlp_tiled(a, st, act, 3, [out])
    bad = [dict(actions=act[:11]), dict(outs=[out[:11]]), dict(state=st.double()),
           dict(actions=torch.zeros(3, 12, device="cuda").t()), dict(state=st.cpu()),
           dict(state=torch.zeros(4, 5, device="cuda")), dict(num_tiled=0)]
    for kw in bad:
        args = dict(arenas=a, state=st, actions=act, num_tiled=3, outs=[out])
        args.update(kw)
        with pytest.raises(AssertionError):
            run_mlp_tiled(**args)
    torch.cuda.synchronize()
