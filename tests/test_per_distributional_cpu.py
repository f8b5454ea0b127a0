"""Prioritized replay for QRDQNTrainer and C51Trainer without a GPU: the weighted oracles against
the reference's QR-DQN and C51 goldens, the row-loss priorities, the C ABI of
rb200_per_priority_update_rows, and FusedDqnStep's argument checks."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import per_distributional_oracle as PD
from oracle import td_oracle as O
from tests import golden_util as G
from tests.golden_cases import C51_CASES, QRDQN_CASES, _c51_kwargs


def _qrdqn_kwargs(meta, batch):
    kw = dict(double_q=meta["double_q"], maxq=meta["maxq"], num_atoms=meta["N"])
    if meta["multi_steps"] is not None:
        kw["discount_src"] = batch["step"]
    return kw


def _check_golden(name, update, kwargs):
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    batch = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = kwargs(meta, batch)
    w = torch.ones(batch["reward"].shape[0])
    for it in range(meta["n_updates"]):
        loss, grads, _ = update(q, qt, adam, batch, w, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(loss - arrays["losses"][it]) <= 1e-6 * max(1.0, abs(arrays["losses"][it]))
        if it == 0:
            for i, g in enumerate(grads):
                assert G.rel_err(g, arrays[f"grad0.{i}"]) < 1e-6, i
    for net, prefix in ((q, "qN"), (qt, "qtN")):
        ps = O.net_params(net)
        for i, (wt, b) in enumerate(G.net_pairs(arrays, prefix)):
            assert G.rel_err(ps[2 * i], wt) < 1e-6 and G.rel_err(ps[2 * i + 1], b) < 1e-6, (prefix, i)


@pytest.mark.parametrize("name", QRDQN_CASES)
def test_weighted_qrdqn_oracle_with_unit_weights_reproduces_reference(name):
    _check_golden(name, PD.weighted_qrdqn_update, _qrdqn_kwargs)


@pytest.mark.parametrize("name", C51_CASES)
def test_weighted_c51_oracle_with_unit_weights_reproduces_reference(name):
    _check_golden(name, PD.weighted_c51_update, _c51_kwargs)


def _toy(B=6, S=5, A=3, N=4, seed=0):
    gen = torch.Generator().manual_seed(seed)
    q = O.make_net([S, 8, A * N], ["relu", "linear"], gen)
    qt = O.clone_net(q)
    batch = {"state": torch.randn(B, S, generator=gen), "next_state": torch.randn(B, S, generator=gen),
             "reward": torch.randn(B, 1, generator=gen), "not_terminal": torch.ones(B, 1),
             "action": torch.eye(A)[torch.arange(B) % A],
             "possible_next_actions_mask": torch.ones(B, A)}
    return q, qt, batch, torch.rand(B, generator=gen) + 0.1


@pytest.mark.parametrize("head", ["qrdqn", "c51"])
def test_weighted_oracles_scale_rows(head):
    """Doubling every weight doubles the loss; a zero weight removes a row's gradient."""
    q, qt, batch, w = _toy()
    N = 4

    def loss_of(weights, b):
        if head == "qrdqn":
            rows, _ = PD.qrdqn_row_loss(q, qt, b, gamma=0.9, num_atoms=N)
        else:
            rows = PD.c51_row_loss(q, qt, b, gamma=0.9, num_atoms=N, qmin=-2.0, qmax=2.0)
        return torch.mean(weights * rows)

    l1, l2 = loss_of(w, batch), loss_of(2 * w, batch)
    assert torch.allclose(l2, 2 * l1, rtol=1e-6, atol=0) and float(l1) > 0
    # the state enters only the current distribution of its own row
    w0 = w.clone()
    w0[2] = 0.0
    state = batch["state"].clone().requires_grad_(True)
    (g,) = torch.autograd.grad(loss_of(w0, dict(batch, state=state)), state)
    assert torch.all(g[2] == 0.0)
    assert all(bool(g[b].abs().sum() > 0) for b in range(g.shape[0]) if b != 2)


def test_row_losses_average_to_the_batch_loss():
    """mean_b(row_b) is td_oracle's batch loss for both heads."""
    q, qt, batch, _ = _toy(seed=3)
    rows, _ = PD.qrdqn_row_loss(q, qt, batch, gamma=0.9, num_atoms=4)
    want, _ = O.qrdqn_loss(q, qt, batch, gamma=0.9, num_atoms=4)
    assert abs(float(rows.mean()) - float(want)) <= 1e-6 * max(1.0, abs(float(want)))
    rows = PD.c51_row_loss(q, qt, batch, gamma=0.9, num_atoms=4, qmin=-2.0, qmax=2.0)
    want = O.c51_loss(q, qt, batch, gamma=0.9, num_atoms=4, qmin=-2.0, qmax=2.0)
    assert abs(float(rows.mean()) - float(want)) <= 1e-6 * max(1.0, abs(float(want)))


def test_row_loss_priorities_known_values():
    p = PD.row_loss_priorities(np.float32([400.0, -100.0, 0.0]), 400.0, 0.5, 1e-6)
    assert np.array_equal(p, np.sqrt(np.array([1.0, 0.25, 0.0]) + 1e-6))
    p = PD.row_loss_priorities(np.float32([2.5]), 1.0, 1.0, 0.0)
    assert p.dtype == np.float64 and p[0] == 2.5
    assert PD.row_loss_priorities(np.float32([3.0]), 1.0, 0.0, 0.0)[0] == 1.0  # alpha 0: uniform


def test_rows_priority_c_abi_rejects_bad_arguments():
    from reagent_b200 import _lib

    lib = _lib.lib()
    x = C.c_void_p(16)  # never dereferenced: the checks reject the call first
    #       tree depth idx row_loss n  divisor alpha eps  p_out max status stream
    good = [x, 3, x, x, 4, 16.0, 0.6, 1e-6, x, x, x, None]
    for pos, name in ((0, "tree"), (2, "idx"), (3, "row_loss"), (8, "p_out"), (10, "status")):
        args = list(good)
        args[pos] = None
        assert lib.rb200_per_priority_update_rows(*args) == -1, name
        err = lib.rb200_last_error()
        assert b"rb200_per_priority_update_rows" in err and name.encode() in err, (name, err)
    for pos, val, what in ((1, -1, b"depth"), (1, 32, b"depth"), (4, 0, b"n"), (4, -3, b"n"),
                           (5, 0.0, b"divisor"), (5, -2.0, b"divisor"),
                           (5, math.inf, b"divisor"), (5, math.nan, b"divisor")):
        args = list(good)
        args[pos] = val
        assert lib.rb200_per_priority_update_rows(*args) == -1, (pos, val)
        err = lib.rb200_last_error()
        assert b"rb200_per_priority_update_rows" in err and what in err, (pos, val, err)


def _cpu_trainers():
    import bench
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.training import C51Trainer

    cfg = dict(bench.CONFIGS[3], S=8, A=3, N=5, B=16, sizes=[8, 8])
    qr = bench.build_trainer(cfg, torch.device("cpu"))
    dist = FullyConnectedDQN(8, 3, [8], ["relu"], num_atoms=5)
    q = CategoricalDQN(dist, qmin=-1.0, qmax=1.0, num_atoms=5)
    c51 = C51Trainer(q, q.get_target_network(), actions=["0", "1", "2"], rl=RLParameters(),
                     num_atoms=5, qmin=-1.0, qmax=1.0)
    return qr, c51


class _Fake:
    """Just enough of a buffer for FusedDqnStep's argument checks, which run first."""
    num_actions = 3


@pytest.mark.parametrize("kw,exc", [
    (dict(rng="host"), ValueError),
    (dict(rng="device", prefetch=True), ValueError),
    (dict(rng="device", shard=(0, 2)), NotImplementedError),
    (dict(rng="device", process_group=object()), NotImplementedError),
])
@pytest.mark.parametrize("which", [0, 1])
def test_fused_step_per_argument_errors_for_distributional_trainers(kw, exc, which):
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    trainer = _cpu_trainers()[which]
    with pytest.raises(exc):
        FusedDqnStep(trainer, _Fake(), 8, per=PrioritizedUpdate(), **kw)


def test_fused_step_per_rejects_other_trainer_types():
    """Only the exact types DQNTrainer, QRDQNTrainer and C51Trainer: a subclass could change
    what the workspace's per-row values mean."""
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training import QRDQNTrainer
    from reagent_b200.training.fused_step import FusedDqnStep

    qr, _ = _cpu_trainers()

    class MyQR(QRDQNTrainer):
        pass

    qr.__class__ = MyQR
    for t in (_Fake(), qr):
        with pytest.raises(NotImplementedError, match="QRDQNTrainer and C51Trainer"):
            FusedDqnStep(t, _Fake(), 8, rng="device", per=PrioritizedUpdate())
