"""Cost of batch-constrained Q-learning (BCQ) in the fused DQN update at config-2 shapes
(B 4096, S 128, A 16, q-network 128-256-128-16 relu, prioritized replay, Huber, double-Q).

BCQ adds two launches before K2 in every update: the imitator's forward on next_state
(rb200_mlp_forward, imitator 128-256-128-16 relu) and rb200_bcq_filter.  This script times, in
one process and alternating the two variants:
  * FusedDqnStep.step() (the whole update as one CUDA graph) with and without BCQ, with the
    replay draws on the host (rng="host") and inside the graph (rng="device"),
  * the imitator forward and rb200_bcq_filter alone, with CUDA events over many launches,
and records the card's name, power limit and maximum SM clock read in the same run.

    python profiles/time_bcq.py --out DIR [--reps 11] [--steps 200]

Writes DIR/time_bcq_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, card_info, cuda_device, host_steps,  # noqa: E402
                             launch_us, write_result)

THRESHOLD = 0.3
CAPACITY = 1 << 18  # replay capacity; per-update time depends on it only through the tree depth


def make_imitator(cfg, dev):
    import torch

    from reagent_b200.models import FullyConnectedNetwork

    torch.manual_seed(1)
    im = FullyConnectedNetwork([cfg["S"]] + list(cfg["sizes"]) + [cfg["A"]],
                               ["relu"] * len(cfg["sizes"]) + ["linear"])
    return im.to(dev)


def build(cfg, dev, bcq, rng):
    import bench
    from reagent_b200.core.parameters import EvaluationParameters, RLParameters
    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training import DQNTrainer
    from reagent_b200.training.dqn_trainer import BCQConfig
    from reagent_b200.training.fused_step import FusedDqnStep
    import torch

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAPACITY, batch_size=cfg["B"],
                                 device=dev)
    rb.add_batch(**bench.synth_stream(CAPACITY, 0, cfg))
    torch.manual_seed(0)
    q = FullyConnectedDQN(cfg["S"], cfg["A"], cfg["sizes"], bench.ACTS)
    kw = dict(imitator=make_imitator(cfg, dev), bcq=BCQConfig(THRESHOLD)) if bcq else {}
    t = DQNTrainer(q.to(dev), q.get_target_network().to(dev),
                   actions=[str(i) for i in range(cfg["A"])],
                   rl=RLParameters(gamma=bench.GAMMA, target_update_rate=bench.TAU,
                                   q_network_loss="huber"),
                   double_q_learning=True, minibatch_size=cfg["B"],
                   optimizer=Optimizer__Union.default(lr=bench.LR),
                   evaluation=EvaluationParameters(calc_cpe_in_training=False), **kw).to(dev)
    return t, FusedDqnStep(t, rb, cfg["B"], rng=rng)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=500)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    import torch

    import bench
    from reagent_b200 import _lib

    cfg = dict(bench.CONFIGS[2])
    info = card_info()
    # rng="host": Python's random stream drawn on the host every step (the default);
    # rng="device": the draws run inside the graph, so the step is bound by the GPU alone
    variants = {f"{k}/rng={rng}": build(cfg, dev, k == "bcq", rng)
                for rng in ("host", "device") for k in ("plain", "bcq")}
    for _, fused in variants.values():
        host_steps(lambda i: fused.step(), args.warmup)
    last_loss = {}

    def run(k, rep):
        us, last_loss[k] = host_steps(lambda i: variants[k][1].step(), args.steps)
        return us

    per_update = alternate(variants, args.reps, run)

    # the two BCQ launches alone, eager, on one sampled batch's next_state
    t = variants["bcq/rng=host"][0]
    B, A = cfg["B"], cfg["A"]
    x = torch.randn(B, cfg["S"], device=dev)
    logits = torch.empty(B, A, device=dev)
    mask = torch.empty(B, A, device=dev)
    im = t.bcq_imitator
    lib, st = _lib.lib(), _lib.cur_stream()

    def imitator_forward():
        _lib.check(lib.rb200_mlp_forward(im.arena.desc(), x.data_ptr(), x.shape[1], None, 0, B,
                                         logits.data_ptr(), None, st), "rb200_mlp_forward")

    def bcq_filter():
        _lib.check(lib.rb200_bcq_filter(logits.data_ptr(), B, A, THRESHOLD, None,
                                        mask.data_ptr(), None, None, st), "rb200_bcq_filter")

    kernels = {"imitator_forward": imitator_forward, "bcq_filter": bcq_filter}
    kern = alternate(kernels, 3, lambda k, rep: launch_us(kernels[k], args.launches))
    dropped = float((mask == 0).float().mean())

    med = {k: v["median"] for k, v in per_update.items()}
    res = {
        "what": ("FusedDqnStep.step() per update, config-2 shapes, with and without BCQ, host "
                 "and device random streams"),
        "card": info,
        "config": dict(B=B, S=cfg["S"], A=A, sizes=cfg["sizes"], replay_capacity=CAPACITY,
                       prioritized=True, imitator=[cfg["S"]] + list(cfg["sizes"]) + [A],
                       drop_threshold=THRESHOLD),
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps; kernels: "
                   f"CUDA events over {args.launches} back-to-back launches after 10 warm-up "
                   f"launches, 3 alternating repetitions"),
        "per_update_us": per_update,
        "bcq_overhead_us_median": {rng: med[f"bcq/rng={rng}"] - med[f"plain/rng={rng}"]
                                   for rng in ("host", "device")},
        "bcq_overhead_frac_median": {rng: med[f"bcq/rng={rng}"] / med[f"plain/rng={rng}"] - 1
                                     for rng in ("host", "device")},
        "kernel_us": {k: dict(median=v["median"], all=v["all"]) for k, v in kern.items()},
        "dropped_fraction_random_states": dropped,
        "last_loss": last_loss,
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
