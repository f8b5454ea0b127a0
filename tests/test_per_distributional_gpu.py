"""Prioritized replay for QRDQNTrainer and C51Trainer on the GPU: importance-weighted
distributional heads against the weighted oracle, the row-loss priorities against numpy and the
host SumTree, and FusedDqnStep(rng="device", online=True, per=...) against a host replica of the
reference buffer, captured and eager."""
import random

import numpy as np
import pytest
import torch

from oracle import per_distributional_oracle as PD
from oracle import td_oracle as O
from tests import golden_util as G
from tests.online_step import (assert_captured_equals_eager, assert_matches_host_replica,
                               assert_nan_reward_raises, bench_setup, filled_heap, params,
                               prioritized_buffer, rows_update, transition_stream, tree, ulps)
from tests.builders import _batch, _build_qr
from tests.golden_cases import C51_CASES, QRDQN_CASES, _c51_kwargs

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _build_c51(meta, arrays):
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import C51Trainer

    S, A, N = meta["S"], meta["A"], meta["N"]
    dist = FullyConnectedDQN(S, A, meta["sizes"], meta["acts"], num_atoms=N)
    G.load_into_module(arrays, "q0", dist)
    q = CategoricalDQN(dist, qmin=meta["qmin"], qmax=meta["qmax"], num_atoms=N)
    qt = q.get_target_network()
    G.load_into_module(arrays, "qt0", qt.distributional_network)
    rl = RLParameters(gamma=meta["gamma"], target_update_rate=meta["tau"], maxq_learning=meta["maxq"],
                      multi_steps=meta["multi_steps"], reward_boost=meta["boost"])
    return C51Trainer(q.cuda(), qt.cuda(), actions=[str(i) for i in range(A)], rl=rl,
                      double_q_learning=meta["double_q"], minibatch_size=meta["B"], num_atoms=N,
                      qmin=meta["qmin"], qmax=meta["qmax"],
                      optimizer=Optimizer__Union.default(lr=meta["lr"])).cuda()


def _golden(name):
    """(trainer, gpu batch, oracle q, oracle qt, cpu batch, oracle kwargs, weighted update,
    divisor D of the head's loss_partials, (q, q_target) modules of the trainer)"""
    arrays, meta = G.load(name)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    cpu = G.batch_tensors(arrays)
    batch = _batch(G.batch_tensors(arrays, "cuda"), meta)
    if name.startswith("qrdqn"):
        t = _build_qr(meta, arrays)
        kw = dict(double_q=meta["double_q"], maxq=meta["maxq"], num_atoms=meta["N"])
        if meta["multi_steps"] is not None:
            kw["discount_src"] = cpu["step"]
        return (t, batch, q, qt, cpu, kw, PD.weighted_qrdqn_update, meta["N"] ** 2,
                (t.q_network, t.q_network_target), meta)
    t = _build_c51(meta, arrays)
    return (t, batch, q, qt, cpu, _c51_kwargs(meta, cpu), PD.weighted_c51_update, 1,
            (t.q_network.distributional_network, t.q_network_target.distributional_network), meta)


@pytest.mark.parametrize("name", ["qrdqn_double", "qrdqn_dueling", "c51_double"])
def test_unit_weights_are_bit_identical_to_unweighted(name):
    out = []
    for weighted in (False, True):
        t, batch, *_, meta = _golden(name)
        w = torch.ones(meta["B"], device="cuda") if weighted else None
        losses, dz = [], []
        for it in range(3):
            losses.append(t.train_batch(batch, it, importance_weights=w).clone())
            dz.append([d.clone() for d in t._ws["net"].dz if d is not None])
        out.append((losses, dz, [p.detach().clone() for p in t.q_network.parameters()],
                    t._ws["loss_partials"].clone()))
    (l0, d0, p0, r0), (l1, d1, p1, r1) = out
    assert all(torch.equal(a, b) for a, b in zip(l0, l1))
    assert all(torch.equal(a, b) for x, y in zip(d0, d1) for a, b in zip(x, y))
    assert all(torch.equal(a, b) for a, b in zip(p0, p1))
    assert torch.equal(r0, r1)


@pytest.mark.parametrize("name", QRDQN_CASES + C51_CASES)
def test_weighted_update_matches_oracle(name):
    """Random weights in [0.05, 1] on the golden batches: loss of every update, the head's
    unweighted per-row losses (loss_partials / D) and the final q and target networks."""
    t, batch, q, qt, cpu, kw, update, D, (qn, qtn), meta = _golden(name)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    gen = torch.Generator().manual_seed(1)
    for it in range(meta["n_updates"]):
        w = 0.05 + 0.95 * torch.rand(meta["B"], generator=gen)
        got = float(t.train_batch(batch, it, importance_weights=w.cuda()))
        want, _, aux = update(q, qt, adam, cpu, w, gamma=meta["gamma"], tau=meta["tau"], **kw)
        assert abs(got - want) <= TOL * max(1.0, abs(want)), (it, got, want)
        rows = aux["rows"] if isinstance(aux, dict) else aux
        got_rows = t._ws["loss_partials"].cpu().double() / D
        assert torch.all((got_rows - rows.double()).abs() <= TOL * rows.double().abs().clamp(min=1.0))
    for net, ref in ((qn, q), (qtn, qt)):
        for a, b in zip(net.parameters(), O.net_params(ref)):
            assert G.rel_err(a.detach().cpu(), b.detach()) < TOL


def test_weighted_qrdqn_config3_matches_chunked_oracle():
    """Config-3 shapes (S 128, A 32, N 200, B 4096, 128-256-128 relu trunk), with the bounds of
    test_qrdqn_config3_full_batch_matches_chunked_oracle."""
    S, A, N, B = 128, 32, 200, 4096
    meta = dict(S=S, A=A, N=N, B=B, sizes=[256, 128], acts=["relu", "relu"], gamma=0.99,
                tau=0.005, maxq=True, multi_steps=None, double_q=True, lr=1e-3, n_updates=1)
    gen = torch.Generator().manual_seed(2)
    q = O.make_net([S, 256, 128, A * N], ["relu", "relu", "linear"], gen)
    qt = O.clone_net(q)
    for w_ in qt["W"]:
        w_.add_(torch.randn(w_.shape, generator=gen) * 0.02)
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = q["W"][i].numpy().copy(), q["b"][i].numpy().copy()
        arrays[f"qt0.W{i}"], arrays[f"qt0.b{i}"] = qt["W"][i].numpy().copy(), qt["b"][i].numpy().copy()
    act = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.05).float()
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen), time_diff=torch.ones(B, 1), step=None,
             not_terminal=nt, action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    w = 0.05 + 0.95 * torch.rand(B, generator=gen)
    t = _build_qr(meta, arrays)
    qo = O.clone_net(q, requires_grad=True)
    params = O.net_params(qo)
    # loss = (1/B) sum_b w_b row_b, accumulated over row chunks
    lo, grads, next_action = 0.0, [torch.zeros_like(p) for p in params], []
    for r0 in range(0, B, 256):
        sub = {k: (v[r0:r0 + 256] if v is not None else None) for k, v in b.items()}
        rows, aux = PD.qrdqn_row_loss(qo, qt, sub, gamma=0.99, num_atoms=N)
        lc = torch.sum(w[r0:r0 + 256] * rows) / B
        for g, gc in zip(grads, torch.autograd.grad(lc, params)):
            g.add_(gc)
        lo += float(lc.detach())
        next_action.append(aux["next_action"])
    gb = _batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    loss = float(t._qr_step(gb, sample_weight=w.cuda()))
    assert abs(loss - lo) <= TOL * max(1.0, abs(lo)), (loss, lo)
    diff = int((t._ws["next_idx"].cpu().long() != torch.cat(next_action)).sum())
    assert diff <= 2, diff
    for i, g in enumerate(t.q_network_grads()):
        G.grad_close(g, grads[i], f"grad {i}")


def test_importance_weights_are_validated():
    t, batch, *_, meta = _golden("qrdqn_double")
    for bad in (torch.ones(meta["B"], dtype=torch.float64, device="cuda"),
                torch.ones(meta["B"] + 1, device="cuda"), torch.ones(meta["B"], 1, device="cuda")):
        with pytest.raises(ValueError, match="importance_weights"):
            t.train_batch(batch, 0, importance_weights=bad)
    t, batch, *_, meta = _golden("c51_double")
    with pytest.raises(ValueError, match="importance_weights"):
        t.train_batch(batch, 0, importance_weights=torch.ones(meta["B"] - 1, device="cuda"))


# ---------------------------------------------------------------------------
# row-loss priorities
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["qrdqn_double", "qrdqn_sarsa_multistep", "c51_double",
                                  "c51_single_masked_boost", "config3_like"])
def test_row_priorities_match_numpy_and_host_tree(name):
    """Priorities from the head's own loss_partials: within 4 fp64 ulp of numpy, and the
    write-back is SumTree.set with exactly those values (host loop, bit for bit).  A NaN row loss
    applies nothing and sets status 3."""
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedUpdate

    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=1000, eps=1e-6)
    if name == "config3_like":  # 4096 rows of QR-sized sums
        row_loss = (torch.rand(4096, device="cuda") * 4e4).contiguous()
        D = 200 * 200
    else:
        t, batch, *_, meta = _golden(name)
        t.train_batch(batch, 0)
        row_loss = t._ws["loss_partials"].clone()
        D = meta["N"] ** 2 if name.startswith("qrdqn") else 1
    n = row_loss.numel()
    rng = np.random.RandomState(n)
    cap = 1 << 14
    heap, depth, _ = filled_heap(cap, rng)
    heap_d = torch.from_numpy(heap).cuda()
    ii = rng.randint(0, cap, n).astype(np.int64)
    ii[::7] = ii[0]  # repeated leaves
    idx = torch.from_numpy(ii).cuda()
    p = torch.empty(n, dtype=torch.float64, device="cuda")
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    dm = torch.tensor([0.0], dtype=torch.float64, device="cuda")
    rows_update(heap_d, depth, idx, row_loss, D, per, p, dm, st)
    want = PD.row_loss_priorities(row_loss.cpu().numpy(), D, per.alpha, per.eps)
    got = p.cpu().numpy()
    assert int(st[0]) == 0 and ulps(got, want).max() <= 4
    h, hm = heap.copy(), np.array([0.0])
    _lib.lib().rb200_sumtree_set_host(h.ctypes.data, depth, ii.ctypes.data, got.ctypes.data, n,
                                      hm.ctypes.data)
    assert np.array_equal(heap_d.cpu().numpy(), h) and float(dm) == hm[0]
    bad = row_loss.clone()
    bad[n // 2] = float("nan")
    before, mbefore = heap_d.clone(), dm.clone()
    rows_update(heap_d, depth, idx, bad, D, per, p, dm, st)
    assert int(st[0]) == 3 and torch.equal(heap_d, before) and torch.equal(dm, mbefore)


# ---------------------------------------------------------------------------
# the online loop
# ---------------------------------------------------------------------------
def _cfg(kind):
    import bench

    return dict(bench.CONFIGS[3], cap=4096, B=256, N=200 if kind == "qrdqn" else 51)


def _setup(kind, base, seed=3):
    import bench
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import C51Trainer

    cfg = _cfg(kind)
    if kind == "qrdqn":
        return bench_setup(cfg, base, seed)
    rb = prioritized_buffer(cfg, base)
    torch.manual_seed(seed)
    S, A, N = cfg["S"], cfg["A"], cfg["N"]
    q = CategoricalDQN(FullyConnectedDQN(S, A, cfg["sizes"], bench.ACTS, num_atoms=N),
                       qmin=-10.0, qmax=10.0, num_atoms=N)
    qt = q.get_target_network()
    rl = RLParameters(gamma=bench.GAMMA, target_update_rate=bench.TAU)
    return rb, C51Trainer(q.cuda(), qt.cuda(), actions=[str(i) for i in range(A)], rl=rl,
                          double_q_learning=True, minibatch_size=cfg["B"], num_atoms=N,
                          qmin=-10.0, qmax=10.0,
                          optimizer=Optimizer__Union.default(lr=bench.LR)).cuda()


@pytest.mark.parametrize("kind", ["qrdqn", "c51"])
def test_online_per_loop_equals_host_replica(kind):
    """The online loop against a host replica; each update's priorities are its rows' own
    losses."""
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg(kind)
    S, A, B = cfg["S"], cfg["A"], cfg["B"]
    base = transition_stream(3000, 3, S, A)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=20, eps=1e-6)
    rb_d, t_d = _setup(kind, base)
    rb_h, _ = _setup(kind, base)
    D = cfg["N"] ** 2 if kind == "qrdqn" else 1
    assert_matches_host_replica(
        lambda: FusedDqnStep(t_d, rb_d, B, rng="device", online=True, per=per), rb_h,
        transition_stream(40, 4, S, A), lambda rb: rb.sample_discrete_dqn_batch(B, A),
        lambda t: PD.row_loss_priorities(t._ws["loss_partials"].cpu().numpy(), D, per.alpha,
                                         per.eps))


@pytest.mark.parametrize("with_per", [False, True])
@pytest.mark.parametrize("kind", ["qrdqn", "c51"])
def test_online_captured_equals_eager(kind, with_per):
    """The same online steps through graph replay and through eager launches of the same
    update from identical starting states: losses, parameters, tree and max priority agree bit
    for bit."""
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg(kind)
    base = transition_stream(3000, 7, cfg["S"], cfg["A"])
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=10, eps=1e-6) if with_per else None

    def setup():
        rb, t = _setup(kind, base)
        random.seed(5)
        return FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=per), None

    assert_captured_equals_eager(
        setup, transition_stream(12, 8, cfg["S"], cfg["A"]), 12,
        lambda f: [params(f.trainer.q_network), params(f.trainer.q_network_target), tree(f)],
        drop_priority=(lambda i: i % 2) if with_per else None)


def test_online_per_qrdqn_nan_reward_raises():
    _online_per_nan_reward_raises("qrdqn")


def test_online_per_c51_nan_reward_raises():
    """C51's projection must keep a NaN target (a clamp with fminf / fmaxf turned it into qmin
    and the step trained on the transition without reporting it)."""
    _online_per_nan_reward_raises("c51")


def _online_per_nan_reward_raises(kind):
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg(kind)
    rb, t = _setup(kind, transition_stream(3000, 5, cfg["S"], cfg["A"]))
    random.seed(1)
    fused = FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=PrioritizedUpdate())
    assert_nan_reward_raises(fused, transition_stream(10, 6, cfg["S"], cfg["A"]))


def test_online_qrdqn_step_after_load_state_dict():
    """Parameters written through torch between steps: the QR-DQN step has no tensor-core images
    to rebuild, and the next replay trains from the loaded parameters."""
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg("qrdqn")
    rb, t = _setup("qrdqn", transition_stream(3000, 9, cfg["S"], cfg["A"]))
    random.seed(2)
    fused = FusedDqnStep(t, rb, cfg["B"], rng="device", online=True)
    extra = transition_stream(3, 10, cfg["S"], cfg["A"])
    fused.step({k: v[0] for k, v in extra.items()})
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in t.q_network.state_dict().items()}
    fused.step({k: v[1] for k, v in extra.items()})
    torch.cuda.synchronize()
    t.q_network.load_state_dict(sd)
    before = [p.detach().clone() for p in t.q_network.parameters()]
    out = fused.step({k: v[2] for k, v in extra.items()})
    torch.cuda.current_stream().synchronize()
    assert np.isfinite(float(out[0]))
    assert any(not torch.equal(a, b) for a, b in zip(before, t.q_network.parameters()))
