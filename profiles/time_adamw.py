"""What AdamW and AMSGrad cost in the fused optimizer kernel (K3, adam_soft_kernel).
One process; records the card's name, power limit and maximum SM clock read in the same run.

  a. K3 alone for Adam, AdamW and AdamW + AMSGrad on the q-network arena of bench.py's config 2
     (DQN 128-256-128-16) and config 3 (QR-DQN 128-256-128-6400), with the Polyak update of the
     target arena and 16 split-K gradient slabs (B 4096 / 256 rows per slab).  Timed with CUDA
     events around one replay of a graph of --launches back-to-back K3 launches, so the window
     holds no host enqueue.  AMSGrad reads and writes max_exp_avg_sq: 8 more bytes per
     parameter per step.
  b. The captured QR-DQN online step at config 3 (FusedDqnStep(rng="device", online=True): add
     one transition, draw, update, all in one graph replay) with Adam against AdamW + AMSGrad,
     --steps steps per run, CUDA events around the loop.

Every variant is repeated --reps times in alternating order and the median is reported.

    python profiles/time_adamw.py --out DIR [--reps 11] [--launches 200] [--steps 100]

Writes DIR/time_adamw.json and prints the same JSON.
"""
import argparse
import json
import os
import random
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.time_k2 import card_info  # noqa: E402

OPTIMIZERS = {"adam": ("Adam", {}), "adamw": ("AdamW", {}),
              "adamw_amsgrad": ("AdamW", {"amsgrad": True})}
SPLITS = 16


def _union(name, lr):
    from reagent_b200.optimizer import Optimizer__Union

    member, kw = OPTIMIZERS[name]
    return Optimizer__Union(**{member: dict(kw, lr=lr)})


def k3_graph(cfg, name, launches):
    """A graph of `launches` K3 launches on the config's q-network arena.  Returns (graph,
    number of parameters, what must stay alive with it)."""
    import bench
    import torch

    t = bench.build_trainer(cfg, torch.device("cuda"), seed=0)
    opt = _union(name, bench.LR).make_optimizer_scheduler(t.q_network.parameters())["optimizer"]
    src, tgt = t.q_network.arena, t.q_network_target.arena
    grad = torch.randn(SPLITS, src.n, device="cuda") * 1e-3
    opt.fused_step(target=tgt, tau=bench.TAU, grad=grad)  # warm-up: module load
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(launches):
            opt.fused_step(target=tgt, tau=bench.TAU, grad=grad)
    torch.cuda.synchronize()
    return g, src.n, (t, opt, grad)


def time_graph(g):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3  # us


def online_step(cfg, name):
    import bench
    import torch

    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=cfg["cap"], batch_size=cfg["B"])
    rb.add_batch(**bench.synth_stream(cfg["cap"], 1000, cfg))
    t = bench.build_trainer(cfg, torch.device("cuda"), seed=0)
    t.q_network_optimizer = _union(name, bench.LR)
    t._optimizers_cache = None
    random.seed(1234)
    fused = FusedDqnStep(t, rb, cfg["B"], rng="device", online=True)
    return fused


def time_online(fused, extra, steps):
    import torch

    for i in range(3):
        fused.step({k: v[i] for k, v in extra.items()})
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fused.step({k: v[3 + i] for k, v in extra.items()})
    e1.record()
    e1.synchronize()
    fused.dr.raise_if_failed()
    return e0.elapsed_time(e1) * 1e3 / steps  # us per step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for time_adamw.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    import torch

    import bench

    if not torch.cuda.is_available():
        raise SystemExit("time_adamw.py measures on the GPU; no CUDA device found")
    torch.cuda.set_device(0)
    res = {"card": card_info(), "reps": args.reps, "launches_per_graph": args.launches,
           "split_k_slabs": SPLITS, "k3_alone_us": {}, "online_step_us": {}}

    for c in (2, 3):
        cfg = dict(bench.CONFIGS[c])
        graphs = {n: k3_graph(cfg, n, args.launches) for n in OPTIMIZERS}
        times = {n: [] for n in OPTIMIZERS}
        for _ in range(args.reps):
            for n, (g, _, _) in graphs.items():
                times[n].append(time_graph(g) / args.launches)
        n_params = graphs["adam"][1]
        res["k3_alone_us"][f"config{c}"] = {
            "params": n_params,
            **{n: {"median": statistics.median(v), "min": min(v), "max": max(v)}
               for n, v in times.items()}}
        del graphs
        torch.cuda.empty_cache()

    cfg = dict(bench.CONFIGS[3], cap=1 << 20)
    extra = bench.synth_stream(args.steps + 3, 77, cfg)
    steps = {n: online_step(cfg, n) for n in ("adam", "adamw_amsgrad")}
    times = {n: [] for n in steps}
    for _ in range(args.reps):
        for n, fused in steps.items():
            times[n].append(time_online(fused, extra, args.steps))
    res["online_step_us"]["config3_qrdqn"] = {
        "steps_per_run": args.steps,
        **{n: {"median": statistics.median(v), "min": min(v), "max": max(v)}
           for n, v in times.items()}}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_adamw.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
