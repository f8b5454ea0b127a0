"""Where the time of the fused DQN TD kernel (K2, dqn_td_tc_kernel) goes at config-2 shapes
(B 4096, q-network 128-256-128-16 relu, Huber, double-Q).  One process; records the card's name,
power limit and maximum SM clock read in the same run.

  a. K2 alone at fixed per-CTA work: batch = 32 n rows (n CTAs; every CTA runs the same chain of
     35 weight-ring stages) for n in 1, 8, 32, 64, 128, weights prepacked.  A flat curve over n
     is the per-CTA chain latency; a rising one is contention for a shared resource, such as the
     L2 reads of the weight stream, which every CTA makes for the same ~1 MB.
  b. The captured config-2 step (bench.py's value path: capture_device_only), kernel by kernel
     from a torch.profiler trace of one replay: median duration of the sample kernel (K1), K2,
     the weight-gradient and the Adam kernels, and the idle gap on a stream before each.  Traced
     with the sample kernel of update k+1 on a second stream next to update k (bench.py's
     graph) and with every kernel on one stream, so that K2's duration with and without a
     concurrent K1 can be compared.
  c. The whole captured step per update in both of those arrangements, alternating.

K2 alone is timed with CUDA events around one replay of a graph of --launches back-to-back
launches (no host enqueue in the window), captured after 5 warm-up launches on a side stream;
every variant is repeated --reps times in alternating order, each timed replay after an untimed
one, and the median is reported.

    python profiles/time_k2.py --out DIR [--reps 11] [--launches 200] [--steps 100]

Writes DIR/time_k2_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, capture, card_info, cuda_device,  # noqa: E402
                             replay_us, write_result)

CTAS = (1, 8, 32, 64, 128)
ARRANGEMENTS = {"k1_on_side_stream": True, "one_stream": False}  # capture_device_only overlap


def k2_graph(trainer, rb, rows, A, launches):
    """One eager update at `rows` rows (sizes the trainer's TD workspace and writes the weight
    images), then a graph of `launches` K2 launches on those inputs with the weights prepacked.
    Returns (graph, what must stay alive with it)."""
    from reagent_b200 import _lib

    batch = rb.sample_discrete_dqn_batch(rows, A)
    trainer.train_batch(batch)
    qd, qtd, a, wsc, keep, pack = trainer._last_td_call
    assert pack is not None, "config-2 shapes run K2 on the wgmma path"
    alive = (trainer._ws, keep, batch, pack)
    lib = _lib.lib()

    def launch():
        _lib.check(lib.rb200_dqn_td_step_tc(qd, qtd, a, wsc, pack.data_ptr(), pack.numel(), 1,
                                            _lib.cur_stream()), "rb200_dqn_td_step_tc")

    return capture(launch, launches), alive


def draw(rb, n, B, dev):
    import numpy as np
    import torch

    out = np.empty((n, B), dtype=np.float64)
    for i in range(n):
        qv, pos, _ = rb.host_queries(B)
        while pos:  # retry-free draws only, as bench.py's value path
            qv, pos, _ = rb.host_queries(B)
        out[i] = qv
    return torch.from_numpy(out).to(dev)


def kernel_class(name):
    if "dqn_td_tc" in name:
        return "K2"
    if "wgrad" in name:
        return "wgrad"
    if "adam" in name:
        return "adam"
    if "sample" in name or "draw" in name:
        return "K1"
    return "other"


def breakdown(g, steps, tmp, tag):
    """torch.profiler trace of one replay of a captured `steps`-update graph: per kernel class
    the median duration, and on each stream the median idle gap before a kernel of the class."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    g.replay()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.replay()
        torch.cuda.synchronize()
    path = os.path.join(tmp, f"k2_{tag}.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"]
              if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])
    dur, gap, last_end = {}, {}, {}
    for e in ev:
        c = kernel_class(e["name"])
        s = e.get("args", {}).get("stream", -1)
        dur.setdefault(c, []).append(e["dur"])
        if s in last_end:
            gap.setdefault(c, []).append(e["ts"] - last_end[s])
        last_end[s] = e["ts"] + e["dur"]
    k2 = [e["ts"] for e in ev if kernel_class(e["name"]) == "K2"]
    period = [b - a for a, b in zip(k2, k2[1:])]
    return {
        "kernels_per_update": {c: len(v) / steps for c, v in dur.items()},
        "names": sorted({e["name"][:120] for e in ev}),
        "median_us": {c: statistics.median(v) for c, v in dur.items()},
        "median_gap_before_on_same_stream_us": {c: statistics.median(v) for c, v in gap.items()},
        "median_k2_start_to_start_us": statistics.median(period) if period else None,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    import torch

    import bench
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import capture_device_only

    cfg = dict(bench.CONFIGS[2])
    B, A = cfg["B"], cfg["A"]
    info = card_info()
    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=cfg["cap"], batch_size=B, device=dev)
    rb.add_batch(**bench.synth_stream(cfg["cap"], 1000, cfg))
    trainer = bench.build_trainer(cfg, dev)

    # ---- a: K2 alone, one graph per CTA count ----
    graphs, alive = {}, []
    for n in CTAS:
        graphs[n], keep = k2_graph(trainer, rb, 32 * n, A, args.launches)
        alive.append(keep)
    k2 = alternate(CTAS, args.reps, lambda n, rep: replay_us(graphs[n], args.launches))
    del graphs
    sweep = {str(n): {s: v[s] for s in ("median", "min", "max")} for n, v in k2.items()}

    # ---- b + c: the captured step, K1 next to the update or in line with it ----
    for _ in range(3):  # eager updates first: workspaces and weight images outside the capture
        trainer.train_batch(rb.sample_discrete_dqn_batch(B, A))
    torch.cuda.synchronize()
    steps = {k: capture_device_only(trainer, rb, B, args.steps, draw(rb, args.steps, B, dev),
                                    overlap_sampling=ov) for k, ov in ARRANGEMENTS.items()}
    per_update = alternate(steps, args.reps, lambda k, rep: replay_us(steps[k], args.steps))
    with tempfile.TemporaryDirectory() as tmp:
        traced = {k: breakdown(g, args.steps, tmp, k) for k, g in steps.items()}

    one, full = sweep["1"]["median"], sweep[str(CTAS[-1])]["median"]
    res = {
        "what": ("dqn_td_tc_kernel (K2) at config-2 shapes: alone at 32 rows per CTA over a "
                 "sweep of CTA counts; the captured config-2 step kernel by kernel and per "
                 "update, with the sample kernel (K1) of the next update on a second stream "
                 "(bench.py's graph) and with all kernels on one stream"),
        "card": info,
        "config": dict(B=B, S=cfg["S"], A=A, sizes=cfg["sizes"], double_q=True, loss="huber"),
        "method": (f"K2: CUDA events around one replay of a graph of {args.launches} launches "
                   f"(weights prepacked), captured after 5 warm-up launches on a side stream, "
                   f"{args.reps} alternating repetitions, medians; step: CUDA events around one "
                   f"replay of a {args.steps}-update capture_device_only graph, {args.reps} "
                   f"alternating repetitions; every timed replay after an untimed one; "
                   f"breakdown: torch.profiler (CUDA activities) over one replay of the same "
                   f"graphs, in a separate pass"),
        "k2_alone_us_by_ctas": sweep,
        "k2_128_over_1_cta": full / one,
        "step_per_update_us": per_update,
        "step_breakdown": traced,
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
