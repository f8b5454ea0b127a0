"""Prioritized replay under data parallel on the GPU: the priority exchange followed by the
PER-semantics tree update against the single-GPU write-backs, and FusedDqnStep /
FusedPolicyStep sharded over one process per GPU (world 2 is skipped with fewer GPUs) against
a host replica of the reference buffer, across ranks, and against a single-GPU step."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch
from tests.builders import _free_port
from tests.online_step import (assert_captured_equals_eager, assert_matches_host_replica,
                               bench_setup, drawn_indices, filled_heap, online_steps, params,
                               prioritized_buffer, same_bits, transition_stream, tree, ulps)

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------
# the exchange of a world of one, then the tree update
# ---------------------------------------------------------------------------
def _sources(source, n, rng, nan_at=None):
    td = torch.from_numpy(rng.randn(n).astype(np.float32)).cuda()
    qs = td + torch.from_numpy((3 * rng.randn(n)).astype(np.float32)).cuda()
    loss = torch.from_numpy(rng.exponential(2.0, n).astype(np.float32)).cuda()
    if nan_at is not None:
        (loss if source == "rows" else td)[nan_at] = float("nan")
    return td, qs, loss


@pytest.mark.parametrize("nan", [False, True])
@pytest.mark.parametrize("n", [37, 5000])
@pytest.mark.parametrize("source", ["td", "rows"])
def test_world_one_exchange_then_apply_equals_priority_update(source, n, nan):
    """rb200_per_priority_exchange (world 1) + rb200_per_priority_apply against
    rb200_per_priority_update[_rows]: tree, max_recorded, priorities and status bit for bit --
    past the 4096-set chunk, with repeated leaves, and with a non-finite value (status 3,
    nothing applied)."""
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedUpdate

    per = PrioritizedUpdate(alpha=0.6, eps=1e-6)
    D = 40000.0 if source == "rows" else 1.0
    rng = np.random.RandomState(n + 2 * nan)
    cap = 1 << 14
    heap, depth, mx = filled_heap(cap, rng)
    idx_h = rng.randint(0, cap, n).astype(np.int64)
    idx_h[::7] = idx_h[1]
    idx = torch.from_numpy(idx_h).cuda()
    td, qs, loss = _sources(source, n, rng, nan_at=n // 2 if nan else None)
    lib = _lib.lib()
    runs = []
    for path in ("single", "exchange"):
        t = torch.from_numpy(heap).cuda()
        dm = torch.from_numpy(mx).cuda()
        st = torch.zeros(2, dtype=torch.int32, device="cuda")
        p = torch.full((n,), -1.0, dtype=torch.float64, device="cuda")
        if path == "single" and source == "td":
            _lib.check(lib.rb200_per_priority_update(
                t.data_ptr(), depth, idx.data_ptr(), td.data_ptr(), qs.data_ptr(), n, per.alpha,
                per.eps, p.data_ptr(), dm.data_ptr(), st.data_ptr(), _lib.cur_stream()))
        elif path == "single":
            _lib.check(lib.rb200_per_priority_update_rows(
                t.data_ptr(), depth, idx.data_ptr(), loss.data_ptr(), n, D, per.alpha, per.eps,
                p.data_ptr(), dm.data_ptr(), st.data_ptr(), _lib.cur_stream()))
        else:
            a = _lib.PerExchangeArgsT()
            if source == "td":
                a.td_target, a.q_selected = td.data_ptr(), qs.data_ptr()
            else:
                a.row_loss, a.divisor = loss.data_ptr(), D
            a.alpha, a.eps = per.alpha, per.eps
            a.n_local, a.row0, a.B_global, a.world, a.rank = n, 0, n, 1, 0
            a.out = p.data_ptr()
            _lib.check(lib.rb200_per_priority_exchange(a, _lib.cur_stream()))
            _lib.check(lib.rb200_per_priority_apply(
                t.data_ptr(), depth, idx.data_ptr(), p.data_ptr(), n, dm.data_ptr(),
                st.data_ptr(), _lib.cur_stream()))
        torch.cuda.synchronize()
        runs.append((t, dm, p, st))
    (t0, dm0, p0, st0), (t1, dm1, p1, st1) = runs
    assert same_bits([t0, dm0, p0, st0], [t1, dm1, p1, st1])
    assert int(st0[0]) == (3 if nan else 0)
    if nan:
        assert torch.equal(t0.cpu(), torch.from_numpy(heap))
    else:
        assert not torch.equal(t0.cpu(), torch.from_numpy(heap))


def test_world_one_exchange_writes_its_rows_only():
    """A world of one writes rows [row0, row0 + n_local) of out and nothing else."""
    from reagent_b200 import _lib

    td = torch.randn(100, device="cuda")
    qs = torch.randn(100, device="cuda")
    out = torch.full((300,), 7.0, dtype=torch.float64, device="cuda")
    a = _lib.PerExchangeArgsT()
    a.td_target, a.q_selected, a.out = td.data_ptr(), qs.data_ptr(), out.data_ptr()
    a.alpha, a.eps = 0.5, 0.25
    a.n_local, a.row0, a.B_global, a.world, a.rank = 100, 150, 300, 1, 0
    _lib.check(_lib.lib().rb200_per_priority_exchange(a, _lib.cur_stream()))
    torch.cuda.synchronize()
    want = ((qs - td).abs().double() + 0.25).sqrt()
    assert ulps(out[150:250].cpu().numpy(), want.cpu().numpy()).max() <= 4
    assert bool((out[:150] == 7.0).all()) and bool((out[250:] == 7.0).all())


def test_sharded_step_of_one_rank_equals_the_unsharded_step():
    """FusedDqnStep(per, shard=(0, 1)) -- importance weights of the whole draw, exchange of a
    world of one, PER-semantics tree update -- equals the unsharded step bit for bit over 20
    online steps."""
    import bench
    from reagent_b200.replay_memory import PrioritizedUpdate
    from reagent_b200.training.fused_step import FusedDqnStep

    cfg = dict(bench.CONFIGS[2], cap=4096, B=256)
    base = transition_stream(3000, 7, cfg["S"], cfg["A"])
    extra = transition_stream(20, 8, cfg["S"], cfg["A"])
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=10, eps=1e-6)
    runs = []
    for shard in (None, (0, 1)):
        rb, t = bench_setup(cfg, base)
        random.seed(5)
        fused = FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=per, shard=shard)
        assert fused._shard is None if shard is None else fused._shard.batch_global == cfg["B"]
        losses = list(online_steps(fused, extra, 20, True, drop_priority=lambda i: i % 2))
        runs.append([losses, params(t.q_network), tree(fused), fused.priorities.clone(),
                     fused.weights.clone()])
    assert same_bits(runs[0], runs[1])


# ---------------------------------------------------------------------------
# one process per GPU
# ---------------------------------------------------------------------------
ALGOS = ["dqn", "qrdqn", "c51", "sac", "td3"]


def _cfg(algo):
    import bench

    c = {"dqn": 2, "qrdqn": 3, "c51": 3, "sac": 4, "td3": 5}[algo]
    cfg = dict(bench.CONFIGS[c], cap=4096, B=256)
    if algo == "qrdqn":
        cfg["N"] = 51
    return cfg


def _setup(algo, cfg, base, seed=3):
    """(prioritized buffer, trainer) for algo; C51 on bench's QR-DQN network shapes."""
    import bench
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import C51Trainer

    if algo != "c51":
        return bench_setup(cfg, base, seed)
    rb = prioritized_buffer(cfg, base)
    torch.manual_seed(seed)
    S, A, N = cfg["S"], cfg["A"], 51
    q = CategoricalDQN(FullyConnectedDQN(S, A, cfg["sizes"], bench.ACTS, num_atoms=N),
                       qmin=-10.0, qmax=10.0, num_atoms=N)
    rl = RLParameters(gamma=bench.GAMMA, target_update_rate=bench.TAU)
    return rb, C51Trainer(q.cuda(), q.get_target_network().cuda(),
                          actions=[str(i) for i in range(A)], rl=rl, double_q_learning=True,
                          minibatch_size=cfg["B"], num_atoms=N, qmin=-10.0, qmax=10.0,
                          optimizer=Optimizer__Union.default(lr=bench.LR)).cuda()


def _stream(algo, cfg, n, seed):
    if algo in ("sac", "td3"):
        return transition_stream(n, seed, cfg=cfg)
    return transition_stream(n, seed, cfg["S"], cfg["A"])


def _make(algo, cfg, rb, t, per, shard=None, pg=None):
    from reagent_b200.training.fused_step import FusedDqnStep, FusedPolicyStep

    if algo in ("sac", "td3"):
        A = cfg["A"]
        return FusedPolicyStep(t, rb, cfg["B"], -np.ones(A, np.float32), np.ones(A, np.float32),
                               online=True, per=per, shard=shard, process_group=pg)
    return FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=per, shard=shard,
                        process_group=pg)


def _sampler(algo, cfg):
    B, A = cfg["B"], cfg["A"]
    if algo in ("sac", "td3"):
        lo, hi = -np.ones(A, np.float32), np.ones(A, np.float32)
        return lambda rb: rb.sample_policy_network_batch(B, lo, hi)
    return lambda rb: rb.sample_discrete_dqn_batch(B, A)


def _digest(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy()).tobytes())
    return h.hexdigest()


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


def _param_bounds(t_dp, t_full):
    """test_dp_gpu.py's measure: worst relative difference, and the fraction above 1e-5."""
    worst = frac = 0.0
    for a, b in zip(t_dp.parameters(), t_full.parameters()):
        scale = float(b.abs().max()) + 1e-30
        d = (a.detach().double() - b.detach().double()).abs()
        worst = max(worst, float(d.max()) / scale)
        frac = max(frac, float((d > 1e-5 * scale).double().mean()))
    return worst, frac


def _worker(rank, world, port, algo, use_p2p, out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        from reagent_b200.replay_memory import PrioritizedUpdate
        from reagent_b200.training.data_parallel import enable_p2p

        pg = dist.group.WORLD
        if use_p2p:
            enable_p2p(pg)
        shard = (rank, world)
        cfg = _cfg(algo)
        base = _stream(algo, cfg, 3000, 3)
        extra = _stream(algo, cfg, 40, 4)
        per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=20, eps=1e-6)
        res = {}

        # (1) a host replica draws the same global indices, takes the gathered priorities and
        # ends with the rank's tree; then every rank holds the same tree, MT state, parameters
        rb_d, t_d = _setup(algo, cfg, base)
        rb_h, _ = _setup(algo, cfg, base)
        torch.manual_seed(17)
        fused = assert_matches_host_replica(lambda: _make(algo, cfg, rb_d, t_d, per, shard, pg),
                                            rb_h, extra, _sampler(algo, cfg), steps=12)
        mine = _digest(fused.rb.sum_tree.heap, [fused.rb.sum_tree.max_recorded_priority],
                       np.asarray(random.getstate()[1], np.int64), *list(t_d.parameters()))
        every = [None] * world
        dist.all_gather_object(every, mine, group=pg)
        res["ranks_agree"] = len(set(every)) == 1

        # (2) against one GPU on the whole batch from the same seeds: the warm-up update's
        # importance weights, its priorities, and the parameters after 2 updates
        runs = {}
        for which, sh, g in (("dp", shard, pg), ("one", None, None)):
            rb, t = _setup(algo, cfg, base)
            random.seed(5)
            torch.manual_seed(23)
            f = _make(algo, cfg, rb, t, per, sh, g)
            torch.cuda.synchronize()
            w, p = f.weights.clone(), f.priorities.clone()
            f.step({k: v[0] for k, v in extra.items()})
            torch.cuda.synchronize()
            runs[which] = (t, w, p, drawn_indices(f))
        (t_dp, w_dp, p_dp, i_dp), (t_one, w_one, p_one, i_one) = runs["dp"], runs["one"]
        res["same_draw"] = bool(np.array_equal(i_dp, i_one))
        res["weights_bits"] = same_bits(w_dp, w_one)
        res["priorities_rel"] = _rel(p_dp, p_one)
        res["params"] = _param_bounds(t_dp, t_one)

        # (3) SAC / TD3 without per: the mean of the ranks' shard losses is the full-batch loss
        if algo in ("sac", "td3"):
            losses = {}
            for which, sh, g in (("dp", shard, pg), ("one", None, None)):
                rb, t = _setup(algo, cfg, base)
                random.seed(5)
                torch.manual_seed(29)
                f = _make(algo, cfg, rb, t, None, sh, g)
                loss = f.step({k: v[0] for k, v in extra.items()})
                torch.cuda.synchronize()
                losses[which] = loss.clone().to(dev)
            dist.all_reduce(losses["dp"], group=pg)
            res["loss_rel"] = _rel(losses["dp"] / world, losses["one"])

        # (4) captured equals eager on this rank
        def setup():
            rb, t = _setup(algo, cfg, base)
            random.seed(5)
            torch.manual_seed(31)
            return _make(algo, cfg, rb, t, per, shard, pg), None

        assert_captured_equals_eager(setup, extra, 6,
                                     lambda f: [params(f.trainer), tree(f), f.priorities],
                                     drop_priority=lambda i: i % 2, scalar_loss=False)
        res["captured_eager"] = True

        # (5) a NaN reward drawn by the next update raises on every rank at the same step
        rb, t = _setup(algo, cfg, _stream(algo, cfg, 3000, 5))
        random.seed(1)
        f = _make(algo, cfg, rb, t, PrioritizedUpdate(), shard, pg)
        bad = {k: v[0] for k, v in extra.items()}
        bad["reward"] = np.float32("nan")
        bad["priority"] = 1e9
        raised_at = -1
        for i in range(10):  # each step completes before the next reads its status
            try:
                f.step(bad if i == 0 else {k: v[i] for k, v in extra.items()})
            except FloatingPointError:
                raised_at = i
                break
            torch.cuda.current_stream().synchronize()
        torch.cuda.synchronize()
        every = [None] * world
        dist.all_gather_object(every, raised_at, group=pg)
        res["nan_steps"] = every
        out.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("use_p2p", [True, False])
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("world", [1, 2])
def test_sharded_prioritized_step(world, algo, use_p2p):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, algo, use_p2p, out))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = [out.get(timeout=1100) for _ in range(world)]
        for p in procs:
            p.join(60)
            assert p.exitcode == 0, f"worker exit code {p.exitcode}"
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    for rank, r in res:
        assert r["ranks_agree"], rank
        assert r["same_draw"] and r["weights_bits"], rank
        assert r["priorities_rel"] <= 1e-5, (rank, r["priorities_rel"])
        worst, frac = r["params"]
        assert worst < 0.05 and frac < 2e-3, (rank, worst, frac)
        if "loss_rel" in r:
            assert r["loss_rel"] <= 1e-5, (rank, r["loss_rel"])
        assert r["captured_eager"]
        steps = r["nan_steps"]
        assert len(set(steps)) == 1 and steps[0] > 0, (rank, steps)
