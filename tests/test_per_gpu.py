"""Prioritized replay on the GPU (FusedDqnStep(per=...)): importance-weighted K2 against the
oracle, the ordered batched SumTree.set against the sequential host loop, the priority / weight
kernels against numpy, and an online loop against a host replica of the reference buffer."""
import random

import numpy as np
import pytest
import torch

from oracle import bcq_oracle as BO
from oracle import per_oracle as P
from oracle import td_oracle as O
from tests import golden_util as G
from tests.online_step import (assert_captured_equals_eager, assert_matches_host_replica,
                               assert_nan_reward_raises, bench_setup, filled_heap, params,
                               transition_stream, tree, ulps)
from tests.builders import (CONFIG2_DZ_TOL, CONFIG2_MAX_ADAM_OUTLIER_FRAC, CONFIG2_MAX_FLIPPED_ROWS,
                            K2_PATHS, _assert_k2, _build_bcq, _build_cpe_trainer, _build_trainer,
                            _golden_batch, _rlt_batch, _select_k2)
from tests.golden_cases import BCQ_DQN_CASES, DQN_CPE_CASES, _dqn_kwargs
from tests.golden_util import TOL

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("path", K2_PATHS)
def test_unit_weights_are_bit_identical_to_unweighted(path, monkeypatch):
    _select_k2(monkeypatch, path)
    arrays, meta = G.load("dqn_huber_double")
    out = []
    for weighted in (False, True):
        t = _build_trainer(meta, arrays)
        batch = _rlt_batch(G.batch_tensors(arrays, "cuda"), meta)
        w = torch.ones(meta["B"], device="cuda") if weighted else None
        losses, dz = [], []
        for it in range(3):
            losses.append(t.train_batch(batch, it, importance_weights=w).clone())
            dz.append([d.clone() for d in t._ws["net"].dz if d is not None])
        _assert_k2(t, path)
        out.append((losses, dz, [p.detach().clone() for p in t.q_network.parameters()]))
    (l0, d0, p0), (l1, d1, p1) = out
    assert all(torch.equal(a, b) for a, b in zip(l0, l1))
    assert all(torch.equal(a, b) for x, y in zip(d0, d1) for a, b in zip(x, y))
    assert all(torch.equal(a, b) for a, b in zip(p0, p1))


WEIGHTED_CASES = (["dqn_huber_double", "dqn_mse_single_masked", "dqn_multistep_boost",
                   "dqn_timediff_odd_dims"] + BCQ_DQN_CASES + DQN_CPE_CASES)


@pytest.mark.parametrize("path", K2_PATHS)
@pytest.mark.parametrize("name", WEIGHTED_CASES)
def test_weighted_update_matches_oracle(name, path, monkeypatch):
    """Random weights in [0.05, 1] on the golden batches, with BCQ and with the CPE heads: the
    TD loss and the q-networks follow the weighted oracle; the CPE losses and networks follow the
    oracle's UNWEIGHTED CPE update (evaluated, as in the reference, after the q-network step)."""
    _select_k2(monkeypatch, path)
    arrays, meta = G.load(name)
    bcq = meta.get("bcq") is not None
    cpe = meta.get("cpe_metrics") is not None
    if bcq:
        t = _build_bcq(meta, arrays)
    elif cpe:
        t = _build_cpe_trainer(meta, arrays)
    else:
        t = _build_trainer(meta, arrays)
    _, batch = _golden_batch(arrays, meta)
    acts = meta["acts"] + ["linear"]
    q = G.oracle_net(arrays, "q0", acts, requires_grad=True)
    qt = G.oracle_net(arrays, "qt0", acts)
    cpu = G.batch_tensors(arrays)
    adam = O.AdamState(O.net_params(q), lr=meta["lr"])
    kw = _dqn_kwargs(meta, cpu)
    if bcq:
        kw.update(imitator=G.oracle_net(arrays, "im", meta["imitator_acts"]),
                  bcq_threshold=meta["bcq"])
    if cpe:
        rn = G.oracle_net(arrays, "r0", acts, requires_grad=True)
        qc = G.oracle_net(arrays, "c0", acts, requires_grad=True)
        qct = G.oracle_net(arrays, "ct0", acts)
        adam_r = O.AdamState(O.net_params(rn), lr=meta["lr"])
        adam_c = O.AdamState(O.net_params(qc), lr=meta["lr"])
        ckw = dict(gamma=meta["gamma"], temperature=meta["temperature"], num_actions=meta["A"],
                   maxq=meta["maxq"], loss=meta["loss"], discount_src=kw.get("discount_src"),
                   imitator=kw.get("imitator"), bcq_threshold=kw.get("bcq_threshold"))
    gen = torch.Generator().manual_seed(1)
    for it in range(meta["n_updates"]):
        w = 0.05 + 0.95 * torch.rand(meta["B"], generator=gen)
        got = float(t.train_batch(batch, it, importance_weights=w.cuda()))
        want, _, _ = P.weighted_dqn_update(q, qt, adam, cpu, w, gamma=meta["gamma"],
                                           tau=meta["tau"], **kw)
        assert abs(got - want) <= 1e-5 * max(1.0, abs(want)), (it, got, want)
        if cpe:
            rl, cl, _, _ = BO.dqn_cpe_update(q, rn, adam_r, qc, qct, adam_c, cpu, tau=meta["tau"],
                                             **ckw)
            for g, wnt in zip((float(x) for x in t.cpe_losses), (rl, cl)):
                assert abs(g - wnt) <= 1e-5 * max(1.0, abs(wnt)), (it, g, wnt)
    _assert_k2(t, path)
    nets = [] if meta.get("dueling") else [(t.q_network, q), (t.q_network_target, qt)]
    if cpe:
        nets += [(t.reward_network, rn), (t.q_network_cpe, qc), (t.q_network_cpe_target, qct)]
    for net, ref in nets:
        for a, b in zip(net.parameters(), O.net_params(ref)):
            assert G.rel_err(a.detach().cpu(), b.detach()) < 1e-5


@pytest.mark.parametrize("path", K2_PATHS)
def test_weighted_config2_matches_oracle(path, monkeypatch):
    """The weighted update at config-2 shapes (S 128, A 16, B 4096, [256, 128] relu, double-Q,
    Huber), with the bounds of test_dqn_config2_matches_oracle: 1e-5 on the rows whose ReLU
    pattern equals the oracle's, a bounded number of flipped rows, and post-Adam elements moved
    by at most the total step size."""
    _select_k2(monkeypatch, path)
    meta = dict(S=128, A=16, B=4096, sizes=[256, 128], acts=["relu", "relu"], gamma=0.99,
                tau=0.005, loss="huber", maxq=True, multi_steps=None, time_diff=False,
                boost=None, double_q=True, lr=1e-3, n_updates=3)
    gen = torch.Generator().manual_seed(0)
    B, S, A = meta["B"], meta["S"], meta["A"]
    q = O.make_net([S, 256, 128, A], ["relu", "relu", "linear"], gen)
    qt = O.clone_net(q)
    for w_ in qt["W"]:
        w_.add_(torch.randn(w_.shape, generator=gen) * 0.02)
    arrays = {}
    for i in range(3):
        arrays[f"q0.W{i}"], arrays[f"q0.b{i}"] = q["W"][i].numpy().copy(), q["b"][i].numpy().copy()
        arrays[f"qt0.W{i}"], arrays[f"qt0.b{i}"] = qt["W"][i].numpy().copy(), qt["b"][i].numpy().copy()
    act = torch.randint(A, (B,), generator=gen)
    nt = (torch.rand(B, 1, generator=gen) > 0.005).float()
    b = dict(state=torch.randn(B, S, generator=gen), next_state=torch.randn(B, S, generator=gen),
             reward=torch.randn(B, 1, generator=gen), time_diff=torch.ones(B, 1), step=None,
             not_terminal=nt, action=torch.nn.functional.one_hot(act, A).float(),
             next_action=torch.nn.functional.one_hot(act, A).float() * nt,
             possible_actions_mask=torch.ones(B, A), possible_next_actions_mask=torch.ones(B, A))
    w = 0.05 + 0.95 * torch.rand(B, generator=gen)
    t = _build_trainer(meta, arrays)
    qo = O.clone_net(q, requires_grad=True)
    adam = O.AdamState(O.net_params(qo), lr=meta["lr"])
    batch = _rlt_batch({k: (v.cuda() if v is not None else None) for k, v in b.items()}, meta)
    okw = dict(double_q=True, maxq=True, loss="huber")

    # per-row view of the first weighted update on the oracle side
    hs, zs = [], []
    x = b["state"]
    for W, bb, a in zip(qo["W"], qo["b"], qo["act"]):
        z = torch.nn.functional.linear(x, W, bb)
        z.retain_grad()
        zs.append(z)
        x = torch.relu(z) if a == "relu" else z
        hs.append(x)
    _, aux = O.dqn_td_loss(qo, qt, b, gamma=meta["gamma"], **okw)
    rows = torch.nn.functional.smooth_l1_loss(torch.sum(hs[-1] * b["action"], 1, keepdim=True),
                                              aux["target"], reduction="none").reshape(-1)
    torch.mean(w * rows).backward()
    dz_ref = [z.grad.detach().clone() for z in zs]
    h_ref = [h.detach() for h in hs]
    for p_ in O.net_params(qo):
        p_.grad = None

    for it in range(meta["n_updates"]):
        lo, grads, aux = P.weighted_dqn_update(qo, qt, adam, b, w, gamma=meta["gamma"],
                                               tau=meta["tau"], **okw)
        got = float(t.train_batch(batch, it, importance_weights=w.cuda()))
        _assert_k2(t, path)
        assert abs(got - lo) <= 2e-5 * max(1.0, abs(lo)), (it, got, lo)
        if it == 0:
            assert G.rel_err(t._ws["td_target"], aux["target"].reshape(-1)) < TOL
            net = t._ws["net"]
            h_gpu = [h.cpu() for h in net.hidden]
            dz_gpu = [z.cpu() for z in net.dz]
            same = torch.ones(B, dtype=torch.bool)
            for l in range(2):
                same &= ((h_gpu[l] > 0) == (h_ref[l] > 0)).all(dim=1)
            assert int((~same).sum()) <= CONFIG2_MAX_FLIPPED_ROWS, int((~same).sum())
            for l in range(3):
                assert G.rel_err(dz_gpu[l][same], dz_ref[l][same]) < CONFIG2_DZ_TOL[path], ("dz", l)
            inputs = [b["state"]] + h_ref[:2]
            g_gpu = t.q_network_grads()
            for l in range(3):
                dzm = dz_ref[l].clone()
                dzm[~same] = dz_gpu[l][~same]
                gw = dzm.double().t() @ inputs[l].double()
                ew = G.rel_err(g_gpu[2 * l], gw)
                eb = G.rel_err(g_gpu[2 * l + 1], dzm.double().sum(0))
                assert ew < CONFIG2_DZ_TOL[path] and eb < CONFIG2_DZ_TOL[path], ("wgrad", l, ew, eb)
    fracs = []
    for i, seq in enumerate(t.q_network.fc.dnn):
        d = (seq[0].weight.detach().cpu().double() - qo["W"][i].detach().double()).abs()
        assert float(d.max()) <= 2.0 * meta["n_updates"] * meta["lr"] * 1.01
        fracs.append(float((d > 1e-5 * float(qo["W"][i].abs().max())).double().mean()))
    assert max(fracs) < CONFIG2_MAX_ADAM_OUTLIER_FRAC, fracs
    for i, seq in enumerate(t.q_network_target.fc.dnn):
        assert G.rel_err(seq[0].weight, qt["W"][i]) < TOL


# ---------------------------------------------------------------------------
# ordered batched SumTree.set
# ---------------------------------------------------------------------------
def _both(heap, depth, mx, idx, val):
    """(host heap, host max, host rc), (device heap, device max, device status)"""
    from reagent_b200 import _lib

    h, hm = heap.copy(), mx.copy()
    idx = np.ascontiguousarray(idx, np.int64)
    val = np.ascontiguousarray(val, np.float64)
    rc = _lib.lib().rb200_sumtree_set_host(h.ctypes.data, depth, idx.ctypes.data, val.ctypes.data,
                                           len(idx), hm.ctypes.data)
    d = torch.from_numpy(heap).cuda()
    dm = torch.from_numpy(mx).cuda()
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    di, dv = torch.from_numpy(idx).cuda(), torch.from_numpy(val).cuda()
    _lib.check(_lib.lib().rb200_sumtree_set_device(
        d.data_ptr(), depth, di.data_ptr(), dv.data_ptr(), len(idx), dm.data_ptr(), st.data_ptr(),
        _lib.cur_stream()), "rb200_sumtree_set_device")
    torch.cuda.synchronize()
    return (h, hm, rc), (d.cpu().numpy(), dm.cpu().numpy(), int(st[0]))


@pytest.mark.parametrize("cap", [64, 1 << 14, 1 << 20])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 4096, 20000])
def test_batched_tree_update_is_bit_equal_to_sequential(n, cap):
    rng = np.random.RandomState(n * 7 + cap)
    heap, depth, mx = filled_heap(cap, rng)
    idx = rng.randint(0, cap, n)
    idx[::5] = idx[0]  # repeated leaves: the order of their sets matters
    val = rng.uniform(0.0, 50.0, n)
    val[1::9] = 0.0
    (h, hm, rc), (d, dm, st) = _both(heap, depth, mx, idx, val)
    assert rc == 0 and st == 0
    assert np.array_equal(d, h) and dm[0] == hm[0]


@pytest.mark.parametrize("case", ["heavy_duplicates", "all_one_leaf", "zeros", "negative_mid"])
def test_batched_tree_update_edge_cases(case):
    rng = np.random.RandomState(11)
    cap, n = 1 << 14, 6000
    heap, depth, mx = filled_heap(cap, rng)
    idx = rng.randint(0, 3, n) * 977
    val = rng.uniform(0.0, 1e3, n)
    if case == "all_one_leaf":
        idx[:] = 5
    elif case == "zeros":
        val[:] = 0.0
        val[::3] = -0.0
    elif case == "negative_mid":
        val[4500] = -1.0  # in the second chunk: the first 4500 sets apply, status 2
    (h, hm, rc), (d, dm, st) = _both(heap, depth, mx, idx, val)
    assert st == (2 if case == "negative_mid" else 0) and rc == (-1 if st else 0)
    assert np.array_equal(d, h)
    assert dm[0] == hm[0] and np.signbit(dm[0]) == np.signbit(hm[0])


# ---------------------------------------------------------------------------
# priority and weight kernels
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("t_frac", [0.0, 0.5, 1.0, 3.0])
def test_priority_and_weight_kernels_match_numpy(t_frac):
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedUpdate

    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=1000, eps=1e-6)
    rng = np.random.RandomState(3)
    cap, B = 1 << 12, 4096
    heap, depth, mx = filled_heap(cap, rng)
    heap_d = torch.from_numpy(heap).cuda()
    idx = torch.from_numpy(rng.randint(0, cap, B).astype(np.int64)).cuda()
    zero_leaf = int(idx[7])
    heap_d[(1 << depth) - 1 + zero_leaf] = 0.0
    step = torch.tensor([int(t_frac * per.beta_updates)], dtype=torch.int64, device="cuda")
    w = torch.empty(B, device="cuda")
    w64 = torch.empty(B, dtype=torch.float64, device="cuda")
    lib = _lib.lib()
    _lib.check(lib.rb200_per_weights(heap_d.data_ptr(), depth, idx.data_ptr(), B, step.data_ptr(),
                                     per.beta0, float(per.beta_updates), w.data_ptr(),
                                     w64.data_ptr(), _lib.cur_stream()))
    leaves = heap_d.cpu().numpy()[(1 << depth) - 1:][idx.cpu().numpy()]
    b = P.beta(int(step), per.beta0, per.beta_updates)
    want = P.importance_weights(leaves, b)
    got = w64.cpu().numpy()
    assert np.all(got[leaves == 0.0] == 0.0) and (leaves == 0.0).any()
    assert ulps(got, want).max() <= 4
    assert np.array_equal(w.cpu().numpy(), got.astype(np.float32))
    # priorities from the device's own TD errors
    td = torch.randn(B, device="cuda")
    qs = td + torch.randn(B, device="cuda") * 3
    p = torch.empty(B, dtype=torch.float64, device="cuda")
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    dm = torch.tensor([0.0], dtype=torch.float64, device="cuda")
    h = heap_d.cpu().numpy().copy()  # the tree before the write-back
    _lib.check(lib.rb200_per_priority_update(heap_d.data_ptr(), depth, idx.data_ptr(), td.data_ptr(),
                                             qs.data_ptr(), B, per.alpha, per.eps, p.data_ptr(),
                                             dm.data_ptr(), st.data_ptr(), _lib.cur_stream()))
    want_p = P.priorities(qs.cpu().numpy(), td.cpu().numpy(), per.alpha, per.eps)
    assert int(st[0]) == 0 and ulps(p.cpu().numpy(), want_p).max() <= 4
    # and the write-back is SumTree.set with exactly those values
    hm = np.array([0.0])
    ii = idx.cpu().numpy()
    pp = p.cpu().numpy()
    lib.rb200_sumtree_set_host(h.ctypes.data, depth, ii.ctypes.data, pp.ctypes.data, B, hm.ctypes.data)
    assert np.array_equal(heap_d.cpu().numpy(), h) and float(dm) == hm[0]
    # a non-finite TD error: nothing applied, status 3
    td[100] = float("nan")
    before = heap_d.clone()
    _lib.check(lib.rb200_per_priority_update(heap_d.data_ptr(), depth, idx.data_ptr(), td.data_ptr(),
                                             qs.data_ptr(), B, per.alpha, per.eps, p.data_ptr(),
                                             dm.data_ptr(), st.data_ptr(), _lib.cur_stream()))
    assert int(st[0]) == 3 and torch.equal(heap_d, before)


# ---------------------------------------------------------------------------
# the online loop against a host replica
# ---------------------------------------------------------------------------
def _cfg():
    import bench

    return dict(bench.CONFIGS[2], cap=4096, B=256)


def test_online_per_loop_equals_host_replica():
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg()
    S, A, B = cfg["S"], cfg["A"], cfg["B"]
    base = transition_stream(3000, 3, S, A)
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=20, eps=1e-6)
    rb_d, t_d = bench_setup(cfg, base)
    rb_h, _ = bench_setup(cfg, base)
    assert_matches_host_replica(
        lambda: FusedDqnStep(t_d, rb_d, B, rng="device", online=True, per=per), rb_h,
        transition_stream(40, 4, S, A), lambda rb: rb.sample_discrete_dqn_batch(B, A))


def test_online_per_captured_equals_eager():
    """The same online steps through graph replay and through eager launches of the same
    update from identical starting states: losses, parameters, tree and max priority agree bit
    for bit."""
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg()
    base = transition_stream(3000, 7, cfg["S"], cfg["A"])
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=10, eps=1e-6)

    def setup():
        rb, t = bench_setup(cfg, base)
        random.seed(5)
        return FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=per), None

    assert_captured_equals_eager(setup, transition_stream(12, 8, cfg["S"], cfg["A"]), 12,
                                 lambda f: [params(f.trainer.q_network), tree(f)],
                                 drop_priority=lambda i: i % 2)


def test_online_per_nan_reward_raises():
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg()
    rb, t = bench_setup(cfg, transition_stream(3000, 5, cfg["S"], cfg["A"]))
    random.seed(1)
    fused = FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=PrioritizedUpdate())
    assert_nan_reward_raises(fused, transition_stream(10, 6, cfg["S"], cfg["A"]))


def test_per_rejects_other_trainers():
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = _cfg()
    rb, t = bench_setup(cfg, transition_stream(3000, 5, cfg["S"], cfg["A"]))

    class NotDqn:
        num_actions = cfg["A"]

    with pytest.raises(NotImplementedError):
        FusedDqnStep(NotDqn(), rb, cfg["B"], rng="device", online=True, per=PrioritizedUpdate())
    with pytest.raises(ValueError):
        FusedDqnStep(t, rb, cfg["B"], rng="device", prefetch=True, per=PrioritizedUpdate())
