"""Prioritized replay (FusedDqnStep(per=...)) without a GPU: the oracle against the reference's
DQN goldens, argument errors, and the C ABI of the new entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import per_oracle as P
from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import BCQ_DQN_CASES, DQN_CASES, _dqn_kwargs


@pytest.mark.parametrize("name", DQN_CASES)
def test_weighted_oracle_with_unit_weights_reproduces_reference(name):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = _dqn_kwargs(meta, batch)
    w = torch.ones(batch["reward"].shape[0])
    for it in range(meta["n_updates"]):
        loss, grads, _ = P.weighted_dqn_update(q, qt, adam, batch, w, gamma=meta["gamma"],
                                               tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = O.net_params(net)
        for i, (wt, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], wt) < 1e-6 and G.rel_err(ps[2 * i + 1], b) < 1e-6


def test_weighted_oracle_scales_rows():
    """Doubling every weight doubles the loss; a zero weight removes a row's gradient."""
    gen = torch.Generator().manual_seed(0)
    q = O.make_net([5, 8, 3], ["relu", "linear"], gen)
    qt = O.clone_net(q)
    B = 6
    batch = {"state": torch.randn(B, 5, generator=gen), "next_state": torch.randn(B, 5, generator=gen),
             "reward": torch.randn(B, 1, generator=gen), "not_terminal": torch.ones(B, 1),
             "action": torch.eye(3)[torch.arange(B) % 3],
             "possible_next_actions_mask": torch.ones(B, 3)}
    w = torch.rand(B, generator=gen)
    l1, _ = P.weighted_td_loss(q, qt, batch, w, gamma=0.9)
    l2, _ = P.weighted_td_loss(q, qt, batch, 2 * w, gamma=0.9)
    assert torch.allclose(l2, 2 * l1)


def test_priority_weight_and_beta_formulas():
    p = P.priorities(np.float32([1.5, -2.0]), np.float32([1.0, 1.0]), 0.6, 1e-6)
    assert np.allclose(p, (np.array([0.5, 3.0]) + 1e-6) ** 0.6, rtol=0, atol=1e-15)
    w = P.importance_weights([4.0, 0.0, 1.0, 2.0], 0.5)
    assert np.allclose(w, [0.5, 0.0, 1.0, 0.5 ** 0.5])
    assert P.beta(0, 0.4, 100) == 0.4
    assert P.beta(50, 0.4, 100) == 0.4 + 0.6 * 50 / 100
    assert P.beta(100, 0.4, 100) == 1.0 and P.beta(10 ** 6, 0.4, 100) == 1.0


@pytest.mark.parametrize("kw", [dict(beta_updates=0), dict(beta_updates=-5), dict(alpha=-0.1),
                                dict(alpha=float("nan")), dict(eps=-1e-6), dict(eps=float("inf")),
                                dict(beta0=-0.1), dict(beta0=1.5)])
def test_prioritized_update_rejects_bad_parameters(kw):
    from reagent_b200.replay_memory import PrioritizedUpdate

    with pytest.raises(ValueError):
        PrioritizedUpdate(**kw)
    PrioritizedUpdate(alpha=0.0, beta0=1.0, eps=0.0, beta_updates=1)  # the edges are accepted


@pytest.mark.parametrize("name", BCQ_DQN_CASES)
def test_weighted_oracle_with_unit_weights_reproduces_bcq_reference(name):
    """With an imitator the weighted oracle applies the BCQ filter: unit weights reproduce the
    reference's BCQ losses."""
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = _dqn_kwargs(meta, batch)
    kw.update(imitator=G.oracle_net(arrays, "im", meta["imitator_acts"]), bcq_threshold=meta["bcq"])
    w = torch.ones(batch["reward"].shape[0])
    for it in range(meta["n_updates"]):
        loss, _, _ = P.weighted_dqn_update(q, qt, adam, batch, w, gamma=meta["gamma"],
                                           tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))


class _Fake:
    """Just enough of a trainer / buffer for FusedDqnStep's argument checks, which run first."""
    num_actions = 2


@pytest.mark.parametrize("kw,exc", [
    (dict(rng="host"), ValueError),
    (dict(rng="device", prefetch=True), ValueError),
    (dict(rng="device", shard=(0, 2)), NotImplementedError),
    (dict(rng="device", process_group=object()), NotImplementedError),
    (dict(rng="device"), NotImplementedError),  # not a DQNTrainer
])
def test_fused_step_per_argument_errors(kw, exc):
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    with pytest.raises(exc):
        FusedDqnStep(_Fake(), _Fake(), 8, per=PrioritizedUpdate(), **kw)


def test_per_c_abi_null_and_size_checks():
    from reagent_b200 import _lib

    lib = _lib.lib()
    x = C.c_void_p(16)  # never dereferenced: the checks reject the call first
    assert lib.rb200_per_weights(None, 3, x, 4, x, 0.4, 10.0, x, None, None) == -1
    assert lib.rb200_per_weights(x, 3, x, 4, None, 0.4, 10.0, x, None, None) == -1
    assert lib.rb200_per_weights(x, 3, x, 4, x, 0.4, 10.0, None, None, None) == -1
    assert lib.rb200_per_weights(x, 3, x, 0, x, 0.4, 10.0, x, None, None) == -1
    assert lib.rb200_per_weights(x, 3, x, 4, x, 0.4, 0.0, x, None, None) == -1
    assert lib.rb200_per_weights(x, 32, x, 4, x, 0.4, 10.0, x, None, None) == -1
    args = [x, 3, x, x, x, 4, 0.6, 1e-6, x, x, x, None]
    assert lib.rb200_per_priority_update(*args[:2], None, *args[3:]) == -1  # idx
    assert lib.rb200_per_priority_update(*args[:3], None, *args[4:]) == -1  # td_target
    assert lib.rb200_per_priority_update(*args[:4], None, *args[5:]) == -1  # q_selected
    assert lib.rb200_per_priority_update(*args[:8], None, *args[9:]) == -1  # p_out
    assert lib.rb200_per_priority_update(*args[:10], None, None) == -1      # status
    assert lib.rb200_per_priority_update(*args[:5], 0, *args[6:]) == -1     # n
    assert b"rb200_per_priority_update" in lib.rb200_last_error()
    a = _lib.AddArgsT()
    a.priority_from_max = 1  # without a tree and max_priority
    st = torch.zeros(4, dtype=torch.int64)
    a.rb.state, a.rb.valid, a.rb.terminal, a.rb.reward = (st.data_ptr(),) * 4
    a.terminal_in = a.reward_in = st.data_ptr()
    a.n, a.rb.capacity, a.rb.update_horizon = 1, 4, 1
    assert lib.rb200_replay_add_device(a, None) == -1
    assert b"priority_from_max" in lib.rb200_last_error()
