"""Host side of ParametricDQN end to end: the ParametricDQN manager's fields and checks, the
trainer's action width, FusedDqnStep's refusals, and the argument checks of
rb200_mlp_forward_tiled (which reject the call before any launch)."""
import ctypes as C

import pytest
import torch
from tests.golden_cases import CARTPOLE_CASES, INPUTMAKER_CASES, cartpole_batch


def test_parametric_dqn_manager_fields():
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.model_managers import ParametricDQN
    from reagent_b200.net_builder import ParametricFullyConnected
    from reagent_b200.optimizer import Optimizer__Union

    m = ParametricDQN()
    assert m.double_q_learning and m.minibatches_per_step == 1
    assert isinstance(m.net_builder, ParametricFullyConnected)
    assert (m.net_builder.sizes, m.net_builder.activations) == ([128, 64], ["relu", "relu"])
    assert type(m.optimizer.value).__name__ == "Adam"
    assert m.eval_parameters == EvaluationParameters()
    assert m.rl_parameters is m.rl
    m = ParametricDQN(rl=RLParameters(maxq_learning=False, temperature=0.35),
                      optimizer=Optimizer__Union(AdamW={"lr": 1e-3, "amsgrad": True}))
    assert m.rl_parameters.temperature == 0.35
    s = {"state": None, "action": None}
    with pytest.raises(RuntimeError):
        m.build_trainer(s, use_gpu=False)


def _trainer():
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.training import ParametricDQNTrainer

    q = FullyConnectedCritic(4, 3, [8], ["relu"])
    return ParametricDQNTrainer(q, q.get_target_network())


def test_trainer_action_width():
    assert _trainer().num_actions == 3


class _Buffer:
    """Enough of a buffer for FusedDqnStep's argument checks, which run first."""


@pytest.mark.parametrize("kw", [dict(per=object(), rng="device", online=True),
                                dict(per=object()), dict(shard=(0, 2)),
                                dict(process_group=object())])
def test_fused_step_refuses_per_and_data_parallel_for_parametric_dqn(kw):
    from reagent_b200.training.fused_step import FusedDqnStep

    with pytest.raises(NotImplementedError):
        FusedDqnStep(_trainer(), _Buffer(), 8, **kw)


def test_tiled_forward_argument_checks():
    from reagent_b200 import _lib
    from reagent_b200.models.arena import ParamArena

    lib = _lib.lib()
    a = ParamArena([9, 16, 1], [1, 0])
    a.flat = torch.zeros(a.n)  # never dereferenced: the checks reject each call first
    b = ParamArena([9, 24, 1], [1, 0])
    b.flat = torch.zeros(b.n)
    x = C.c_void_p(16)

    def call(n0=a.desc(), n1=None, st=x, S=6, act=x, K=3, B=4, M=3, out0=x, out1=None):
        return lib.rb200_mlp_forward_tiled(n0, n1, st, S, act, K, B, M, out0, out1, None)

    for kw in [dict(st=None), dict(act=None), dict(out0=None), dict(n0=None),
               dict(n1=a.desc()), dict(out1=x), dict(n1=b.desc(), out1=x), dict(S=5),
               dict(K=4), dict(S=0, K=9), dict(B=0), dict(M=0), dict(B=-3),
               dict(B=1 << 16, M=1 << 15)]:
        assert call(**kw) == -1, kw
    assert "int32" in lib.rb200_last_error().decode()
    wide = ParamArena([9, 16, 1100], [1, 0])
    wide.flat = torch.zeros(wide.n)
    assert call(n0=wide.desc()) == -3


# ---------------------------------------------------------------------------
# the oracle restatements pinned against the reference's goldens
# (oracle/make_parametric_golden.py)
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("name", INPUTMAKER_CASES)
def test_replay_oracle_plus_parametric_inputmaker_match_reference(name):
    """The oracle sampler followed by ParametricDqnInputMaker's arithmetic (one-hot actions, the
    next one zeroed on terminal rows, 1 - terminal, the identity tiling, ones masks,
    exp(log_prob)) reproduces the reference's batches on the same seeds."""
    import random

    import numpy as np

    from oracle.replay_oracle import ReplayOracle
    from tests import golden_util as G

    arrays, meta = G.load(name)
    ro = ReplayOracle(meta["cap"], update_horizon=meta["horizon"], gamma=meta["gamma"],
                      prioritized=meta["prioritized"])
    st = {k: arrays[f"stream.{k}"] for k in meta["keys"]}
    for t in range(meta["n_add"]):
        ro.add(**{k: v[t] for k, v in st.items()})
    random.seed(meta["seed"] + 200)
    torch.manual_seed(meta["seed"] + 200)
    A, B = meta["A"], meta["B"]
    eye = np.eye(A, dtype=np.float32)
    for s_i in range(meta["n_samples"]):
        ob = ro.sample_transition_batch(B)
        pre = f"sample{s_i}."
        assert np.array_equal(ob["indices"], arrays[pre + "indices"].reshape(-1))
        term = ob["terminal"].astype(bool)
        assert np.array_equal(term, arrays[pre + "terminal"].reshape(-1))
        assert np.array_equal(ob["state"], arrays[pre + "state"])
        assert np.array_equal(ob["next_state"][~term], arrays[pre + "next_state"][~term])
        np.testing.assert_allclose(ob["reward"], arrays[pre + "reward"].reshape(-1), rtol=2e-6,
                                   atol=1e-6)
        assert np.array_equal(1.0 - term.astype(np.float32), arrays[pre + "not_terminal"].reshape(-1))
        assert np.array_equal(eye[ob["action"]], arrays[pre + "action"])
        assert np.array_equal(eye[ob["next_action"]] * (~term)[:, None], arrays[pre + "next_action"])
        tiled = np.tile(eye, (B, 1))
        assert np.array_equal(tiled, arrays[pre + "possible_actions"])
        assert np.array_equal(tiled, arrays[pre + "possible_next_actions"])
        ones = np.ones((B, A), dtype=np.float32)
        assert np.array_equal(ones, arrays[pre + "possible_actions_mask"])
        assert np.array_equal(ones, arrays[pre + "possible_next_actions_mask"])
        lp = torch.from_numpy(np.asarray(ob["log_prob"], dtype=np.float32))
        assert np.array_equal(lp.exp().numpy().reshape(-1),
                              arrays[pre + "action_probability"].reshape(-1))


@pytest.mark.parametrize("name", CARTPOLE_CASES)
def test_pdqn_oracle_matches_reference_cartpole(name):
    """td_oracle.pdqn_update with Adam / AdamW + AMSGrad reproduces the reference trainer as the
    ParametricDQN manager wires it, update by update, and the networks after five updates."""
    from oracle import td_oracle as O
    from oracle.adamw_oracle import AdamWState
    from tests import golden_util as G

    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    rn = G.oracle_net(arrays, "r0", acts, requires_grad=True)

    def opt(net):
        if meta["optimizer"] == "AdamW":
            return AdamWState(O.net_params(net), lr=meta["lr"], weight_decay=meta["weight_decay"],
                              amsgrad=meta["amsgrad"])
        return O.AdamState(O.net_params(net), lr=meta["lr"])

    adam, adam_r = opt(q), opt(rn)
    for it in range(meta["n_updates"]):
        batch = cartpole_batch(arrays, it)
        td, rl, _ = O.pdqn_update(q, qt, adam, batch, gamma=meta["gamma"], tau=meta["tau"],
                                  double_q=meta["double_q"], maxq=meta["maxq"], loss="mse",
                                  reward_net=rn, adam_r=adam_r)
        for got, want in ((td, arrays["losses"][it][0]), (rl, arrays["losses"][it][1])):
            assert abs(got - want) <= 1e-6 * max(1.0, abs(want)), (it, got, want)
    for net, prefix in ((q, "qN"), (qt, "qtN"), (rn, "rN")):
        ps = O.net_params(net)
        for i, (w, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], w) < 1e-6 and G.rel_err(ps[2 * i + 1], b) < 1e-6, (prefix, i)


def test_scorer_restatement_and_softmax_draws_match_reference():
    """q(obs[i] tiled, identity tiling).view(-1, A) restates parametric_dqn_scorer; this
    package's SoftmaxActionSampler on the reference's scores repeats its seeded draws."""
    from oracle import td_oracle as O
    from reagent_b200.gym.policies import SoftmaxActionSampler
    from tests import golden_util as G

    arrays, meta = G.load("parametric_scorer")
    A, n = meta["A"], meta["n"]
    q = G.oracle_net(arrays, "q", meta["acts"] + ["linear"])
    obs = torch.from_numpy(arrays["obs"])
    with torch.no_grad():
        scores = O.critic(q, obs.repeat_interleave(A, dim=0), torch.eye(A).repeat(n, 1)).view(-1, A)
    assert G.rel_err(scores, arrays["scores"]) < 1e-6
    want_scores = torch.from_numpy(arrays["scores"])
    for ti, temp in enumerate(meta["temperatures"]):
        sm = SoftmaxActionSampler(temperature=temp)
        for d in range(meta["n_draws"]):
            torch.manual_seed(meta["seed"] + 100 * (ti + 1) + d)
            out = sm.sample_action(want_scores)
            assert torch.equal(out.action, torch.from_numpy(arrays[f"t{ti}.d{d}.action"]))
            assert torch.equal(out.log_prob, torch.from_numpy(arrays[f"t{ti}.d{d}.log_prob"]))
