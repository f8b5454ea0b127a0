"""N = 2 data-parallel parity on hardware (skipped with fewer than two GPUs): one DP update -- row shards of the same global minibatch, gradient exchange
(a) fused into the Adam kernel over NVLink peer memory and (b) by plain NCCL all-reduce --
against one full-batch update on a single rank from identical parameters.  SURVEY.md 8e: every
loss is a batch mean, so the mean of the shard gradients is the global gradient."""
import os

import pytest
import torch
from tests.builders import _free_port

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, algo, use_p2p, out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        from reagent_b200.core import types as rlt
        from reagent_b200.training.data_parallel import enable_p2p, shard_rows
        import bench

        if use_p2p:
            enable_p2p(dist.group.WORLD)
        cfg = dict(bench.CONFIGS[{"dqn": 2, "sac": 4, "td3": 5}[algo]])
        cfg["B"] = 1024 if algo == "dqn" else 512
        B, S, A = cfg["B"], cfg["S"], cfg["A"]
        lo, hi = shard_rows(B, rank, world)
        g = torch.Generator(device=dev).manual_seed(3)
        r = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
        state, nstate, reward = r(B, S), r(B, S), r(B, 1)
        nt = (torch.rand(B, 1, device=dev, generator=g) > 0.05).float()
        if algo == "dqn":
            act = torch.nn.functional.one_hot(torch.randint(A, (B,), device=dev, generator=g), A).float()

            def mk(sl):
                return rlt.DiscreteDqnInput(
                    state=rlt.FeatureData(state[sl]), next_state=rlt.FeatureData(nstate[sl]),
                    reward=reward[sl], time_diff=None, step=None, not_terminal=nt[sl],
                    action=act[sl], next_action=act[sl] * nt[sl],
                    possible_actions_mask=torch.ones(B, A, device=dev)[sl],
                    possible_next_actions_mask=torch.ones(B, A, device=dev)[sl], extras=rlt.ExtraData())
        else:
            act = torch.rand(B, A, device=dev, generator=g) * 1.98 - 0.99

            def mk(sl):
                return rlt.PolicyNetworkInput(
                    state=rlt.FeatureData(state[sl]), next_state=rlt.FeatureData(nstate[sl]),
                    reward=reward[sl], time_diff=None, step=None, not_terminal=nt[sl],
                    action=rlt.FeatureData(act[sl]), next_action=rlt.FeatureData(act[sl] * nt[sl]),
                    extras=rlt.ExtraData())
        t_dp, t_full = bench.build_trainer(cfg, dev, seed=11), bench.build_trainer(cfg, dev, seed=11)
        if algo != "dqn":
            noise = {k: r(B, A) for k in ("next", "cur")}
            t_full.noise_hook = lambda name, shape, device: noise[name]
            t_dp.noise_hook = lambda name, shape, device: noise[name][lo:hi]
        worst = 0.0
        for it in range(2):  # two updates: the second uses the other buffer parity
            t_full.train_batch(mk(slice(0, B)), it)
            t_dp.train_batch(mk(slice(lo, hi)), it, process_group=dist.group.WORLD)
        torch.cuda.synchronize()
        frac = 0.0
        for a, b in zip(t_dp.parameters(), t_full.parameters()):
            scale = float(b.abs().max()) + 1e-30
            d = (a.detach().double() - b.detach().double()).abs()
            worst = max(worst, float(d.max()) / scale)
            frac = max(frac, float((d > 1e-5 * scale).double().mean()))
        # replicated parameters stay bit-identical across ranks (rank-ordered sums)
        flat = torch.cat([p.detach().reshape(-1) for p in t_dp.parameters()])
        other = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(other, flat)
        same = all(torch.equal(o, flat) for o in other)
        out.put((rank, worst, frac, same))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_p2p", [True, False])
@pytest.mark.parametrize("algo", ["dqn", "sac", "td3"])
def test_two_rank_update_matches_full_batch(algo, use_p2p):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, algo, use_p2p, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(500)
        assert p.exitcode == 0, f"worker exit code {p.exitcode}"
    res = [out.get(timeout=10) for _ in range(2)]
    for rank, worst, frac, same in res:
        # Adam turns gradient elements within fp32 noise of zero into +-lr moves: bounded by the
        # step size, and all but a vanishing fraction within 1e-5
        assert worst < 0.05, (rank, worst)
        assert frac < 2e-3, (rank, frac)
        assert same, "ranks diverged"
