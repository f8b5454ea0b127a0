"""What AdamW and AMSGrad cost in the fused optimizer kernel (K3, adam_soft_kernel).
One process; records the card's name, power limit and maximum SM clock read in the same run.

  a. K3 alone for Adam, AdamW and AdamW + AMSGrad on the q-network arena of bench.py's config 2
     (DQN 128-256-128-16) and config 3 (QR-DQN 128-256-128-6400), with the Polyak update of the
     target arena and 16 split-K gradient slabs (B 4096 / 256 rows per slab).  Timed with CUDA
     events around one replay, after an untimed one, of a graph of --launches back-to-back K3
     launches captured after 5 warm-up launches on a side stream, so the window holds no host
     enqueue.  AMSGrad reads and writes max_exp_avg_sq: 8 more bytes per parameter per step.
  b. The captured QR-DQN online step at config 3 (FusedDqnStep(rng="device", online=True): add
     one transition, draw, update, all in one graph replay) with Adam against AdamW + AMSGrad,
     3 warm-up steps and then --steps steps per run, host-clocked from a synchronise to the
     synchronise after the last step.

Every variant is repeated --reps times, in the given order on even repetitions and reversed on
odd ones, and the median is reported.

    python profiles/time_adamw.py --out DIR [--reps 11] [--launches 200] [--steps 100]

Writes DIR/time_adamw_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, capture, card_info, cuda_device,  # noqa: E402
                             host_steps, replay_us, transitions, write_result)

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
    g = capture(lambda: opt.fused_step(target=tgt, tau=bench.TAU, grad=grad), launches)
    return g, src.n, (t, opt, grad)


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


def time_online(fused, trs, steps):
    host_steps(lambda i: fused.step(trs[i]), 3)
    us, _ = host_steps(lambda i: fused.step(trs[i]), steps, 3)
    fused.dr.raise_if_failed()
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()

    cuda_device(__file__)
    import torch

    import bench

    res = {"card": card_info(), "reps": args.reps, "launches_per_graph": args.launches,
           "split_k_slabs": SPLITS, "k3_alone_us": {}, "online_step_us": {}}

    for c in (2, 3):
        cfg = dict(bench.CONFIGS[c])
        graphs = {n: k3_graph(cfg, n, args.launches) for n in OPTIMIZERS}
        times = alternate(graphs, args.reps,
                          lambda n, rep: replay_us(graphs[n][0], args.launches))
        res["k3_alone_us"][f"config{c}"] = {
            "params": graphs["adam"][1],
            **{n: {s: v[s] for s in ("median", "min", "max")} for n, v in times.items()}}
        del graphs
        torch.cuda.empty_cache()

    cfg = dict(bench.CONFIGS[3], cap=1 << 20)
    trs = transitions(cfg, args.steps + 3, seed=77)
    steps = {n: online_step(cfg, n) for n in ("adam", "adamw_amsgrad")}
    times = alternate(steps, args.reps, lambda n, rep: time_online(steps[n], trs, args.steps))
    res["online_step_us"]["config3_qrdqn"] = {
        "steps_per_run": args.steps,
        **{n: {s: v[s] for s in ("median", "min", "max")} for n, v in times.items()}}
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
