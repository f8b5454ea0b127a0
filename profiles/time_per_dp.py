"""Cost of prioritized replay under data parallel: the captured online step sharded over one
process per GPU, with and without per, and the priority exchange alone.

Shapes: config 2 (DQN, B_global 4096), config 4 (SAC, B_global 8192) and config 5 (TD3,
B_global 16384), each with its bench.py network sizes and a replay capacity of 2^20.  For every
world W in 2, 4 and 8 that the machine has GPUs for, this script spawns W processes (one per
GPU, NCCL group, peer-memory exchange enabled) and times, alternating the variants:
  * captured: FusedDqnStep / FusedPolicyStep(rng="device", online=True, shard=(rank, W),
    process_group=...).step(transition) -- gradients exchanged inside the Adam kernels;
  * captured_per: the same with per=PrioritizedUpdate(): importance weights of the whole draw,
    this rank's weighted rows, and the priorities of all B_global rows exchanged over NVLink
    peer memory and applied to every rank's tree;
  * the exchange kernel alone (rb200_per_priority_exchange at B_global = 4096), CUDA events over
    many back-to-back launches on every rank;
and records the card's name, power limit and maximum SM clock read in the same run.

    python profiles/time_per_dp.py --out DIR [--reps 7] [--steps 100]

Writes DIR/time_per_dp_<card>_<limit>w.json (rank 0's timings) and prints the same JSON.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, card_info, cuda_device, host_steps,  # noqa: E402
                             launch_us, transitions, write_result)

CAPACITY = 1 << 20
CONFIGS = {"dqn": 2, "sac": 4, "td3": 5}


def free_port() -> int:
    import socket

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def build(algo, cfg, dev, stream, per, rank, world, pg):
    import numpy as np

    import bench
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep, FusedPolicyStep

    B = cfg["B"]
    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAPACITY, batch_size=B, device=dev)
    rb.add_batch(**stream)
    t = bench.build_trainer(cfg, dev, seed=0)
    kw = dict(online=True, per=per, shard=(rank, world), process_group=pg)
    if algo == "dqn":
        return FusedDqnStep(t, rb, B, rng="device", **kw)
    low, high = -np.ones(cfg["A"], np.float32), np.ones(cfg["A"], np.float32)
    return FusedPolicyStep(t, rb, B, low, high, **kw)


def worker(rank, world, port, args, out):
    import random

    import numpy as np
    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        import bench
        from reagent_b200 import _lib
        from reagent_b200.replay_memory import PrioritizedUpdate
        from reagent_b200.training.data_parallel import enable_p2p

        pg = dist.group.WORLD
        ex = enable_p2p(pg)
        per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=100_000, eps=1e-6)
        random.seed(1234)
        per_update = {}
        for algo, c in CONFIGS.items():
            cfg = dict(bench.CONFIGS[c])
            stream = bench.synth_stream(CAPACITY, 0, cfg)
            variants = {f"{algo}_captured": build(algo, cfg, dev, stream, None, rank, world, pg),
                        f"{algo}_captured_per": build(algo, cfg, dev, stream, per, rank, world, pg)}
            del stream
            trs = transitions(cfg, 1000)
            for v in variants.values():
                host_steps(lambda i: v.step(trs[i % len(trs)]), args.warmup)

            def run(k, rep):
                return host_steps(lambda i: variants[k].step(trs[i % len(trs)]), args.steps,
                                  rep * args.steps)[0]

            per_update.update(alternate(variants, args.reps, run))
            for v in variants.values():
                v.dr.raise_if_failed()
            del variants
            torch.cuda.synchronize()
            torch.cuda.empty_cache()

        # the exchange alone: B_global = 4096 priorities, this rank's rows from TD errors
        Bg = 4096
        n = Bg // world
        rng = np.random.RandomState(rank)
        td = torch.from_numpy(rng.randn(n).astype(np.float32)).to(dev)
        qs = torch.from_numpy(rng.randn(n).astype(np.float32)).to(dev)
        p = torch.empty(Bg, dtype=torch.float64, device=dev)
        recv, flags, epoch = ex.priority_slice(("time_per_dp", Bg), Bg)
        a = _lib.PerExchangeArgsT()
        a.td_target, a.q_selected, a.out = td.data_ptr(), qs.data_ptr(), p.data_ptr()
        a.alpha, a.eps = per.alpha, per.eps
        a.n_local, a.row0, a.B_global, a.world, a.rank = n, rank * n, Bg, world, rank
        a.recv, a.flags, a.epoch = recv.data_ptr(), flags.data_ptr(), epoch.data_ptr()
        lib, cs = _lib.lib(), _lib.cur_stream()

        def exchange():
            _lib.check(lib.rb200_per_priority_exchange(a, cs))

        xs = []
        for _ in range(3):
            dist.barrier(group=pg)
            xs.append(launch_us(exchange, args.launches))
        torch.cuda.synchronize()
        out.put((rank, per_update, xs))
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    cuda_device(__file__)
    import statistics

    import torch
    import torch.multiprocessing as mp

    n_gpus = torch.cuda.device_count()
    worlds = [w for w in (2, 4, 8) if w <= n_gpus]
    if not worlds:
        raise SystemExit(f"time_per_dp.py needs 2 or more GPUs; {n_gpus} visible")
    info = card_info()
    results = {}
    ctx = mp.get_context("spawn")
    for world in worlds:
        q = ctx.Queue()
        port = free_port()
        procs = [ctx.Process(target=worker, args=(r, world, port, args, q)) for r in range(world)]
        for p in procs:
            p.start()
        try:
            got = dict((r, (u, x)) for r, u, x in (q.get(timeout=3600) for _ in range(world)))
            for p in procs:
                p.join(120)
                if p.exitcode != 0:
                    raise SystemExit(f"world {world}: a worker exited with {p.exitcode}")
        finally:
            for p in procs:
                if p.is_alive():
                    p.kill()
                    p.join()
        per_update, xs = got[0]
        med = {k: v["median"] for k, v in per_update.items()}
        results[f"W{world}"] = {
            "per_update_us_rank0": per_update,
            "per_overhead_us_median": {a: med[f"{a}_captured_per"] - med[f"{a}_captured"]
                                       for a in CONFIGS},
            "exchange_us": {f"rank{r}": dict(median=statistics.median(got[r][1]), all=got[r][1])
                            for r in sorted(got)},
        }
    import bench

    res = {
        "what": ("per update under data parallel (one process per GPU, peer-memory exchange): "
                 "the captured online step with and without per for DQN (config 2), SAC "
                 "(config 4) and TD3 (config 5) at their global batch sizes; the priority "
                 "exchange kernel alone at B_global = 4096"),
        "card": info,
        "gpus_visible": n_gpus,
        "config": {a: dict(B_global=bench.CONFIGS[c]["B"], S=bench.CONFIGS[c]["S"],
                           A=bench.CONFIGS[c]["A"], sizes=bench.CONFIGS[c]["sizes"],
                           replay_capacity=CAPACITY) for a, c in CONFIGS.items()},
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps, each step "
                   f"adding one transition; exchange: CUDA events over {args.launches} "
                   f"back-to-back launches after 10 warm-up launches, 3 repetitions"),
        "worlds": results,
        "timestamp": time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime()),
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
