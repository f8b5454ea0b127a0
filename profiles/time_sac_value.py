"""Cost of SACTrainer's state-value network and CRR weighting.

Shapes: the reference's Pendulum configuration (S 3, A 1, B 256, [64, 64] leaky_relu networks)
and the config-4 per-GPU row (S 256, A 32, B 2048, [256, 256] relu networks), twin critics and a
learnable temperature in both.  This script times, in one process, alternating the variants:
  * train_batch per update without a value network, with one, and with one plus CRR
    (exponent_beta 1, exponent_clamp 20) -- a fixed device-resident batch, host-timed
    synchronised updates;
  * the captured FusedPolicyStep(rng="device", online=True).step() with a value network
    (config-4 shape, replay capacity 2^16);
  * rb200_ac_value_step (ac_value_rows_kernel) alone, CUDA events over many launches;
and records the card's name, power limit and maximum SM clock read in the same run.

    python profiles/time_sac_value.py --out DIR [--reps 11] [--steps 100]

Writes DIR/time_sac_value_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, card_info, cuda_device, host_steps,  # noqa: E402
                             launch_us, transitions, write_result)

SHAPES = {
    "pendulum": dict(S=3, A=1, B=256, sizes=[64, 64], acts=["leaky_relu", "leaky_relu"]),
    "config4": dict(S=256, A=32, B=2048, sizes=[256, 256], acts=["relu", "relu"]),
}
CAPACITY = 1 << 16


def trainer(shape, variant, dev, seed=0):
    import torch

    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic, GaussianFullyConnectedActor
    from reagent_b200.models.fully_connected_network import FloatFeatureFullyConnected
    from reagent_b200.training import CRRWeightFn, SACTrainer

    torch.manual_seed(seed)
    S, A, sz, ac = shape["S"], shape["A"], shape["sizes"], shape["acts"]
    value = None if variant == "no_value" else FloatFeatureFullyConnected(S, 1, sz, ac)
    crr = CRRWeightFn(exponent_beta=1.0, exponent_clamp=20.0) if variant == "crr" else None
    return SACTrainer(GaussianFullyConnectedActor(S, A, sz, ac), FullyConnectedCritic(S, A, sz, ac),
                      FullyConnectedCritic(S, A, sz, ac), value,
                      rl=RLParameters(gamma=0.99, target_update_rate=0.005),
                      minibatch_size=shape["B"], entropy_temperature=0.1,
                      target_entropy=-float(A), crr_config=crr).to(dev)


def batch(shape, dev):
    import torch

    from reagent_b200.core import types as rlt

    g = torch.Generator().manual_seed(1)
    B, S, A = shape["B"], shape["S"], shape["A"]
    f = lambda t: t.to(dev)  # noqa: E731
    return rlt.PolicyNetworkInput(
        state=rlt.FeatureData(f(torch.randn(B, S, generator=g))),
        next_state=rlt.FeatureData(f(torch.randn(B, S, generator=g))),
        action=rlt.FeatureData(f(torch.rand(B, A, generator=g) * 1.98 - 0.99)),
        next_action=rlt.FeatureData(f(torch.zeros(B, A))),
        reward=f(torch.randn(B, 1, generator=g)),
        not_terminal=f((torch.rand(B, 1, generator=g) > 0.01).float()), step=None,
        time_diff=None, extras=rlt.ExtraData())


class TrainLoop:
    def __init__(self, t, b):
        self.t, self.b, self.i = t, b, 0

    def step(self, transition=None):
        closs, _ = self.t.train_batch(self.b, self.i)
        self.i += 1
        return closs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    import random

    import numpy as np
    import torch

    import bench
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedPolicyStep
    from reagent_b200.training.workspace import Pins

    random.seed(1234)
    info = card_info()
    per_update, kernel_us, last_loss = {}, {}, {}
    for sname, shape in SHAPES.items():
        b = batch(shape, dev)
        loops = {f"{sname}_train_batch_{v}": TrainLoop(trainer(shape, v, dev), b)
                 for v in ("no_value", "value", "crr")}
        if sname == "config4":
            cfg = dict(bench.CONFIGS[4], B=shape["B"])
            rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAPACITY,
                                         batch_size=shape["B"], device=dev)
            rb.add_batch(**bench.synth_stream(CAPACITY, 0, cfg))
            low, high = -np.ones(shape["A"], np.float32), np.ones(shape["A"], np.float32)
            loops[f"{sname}_captured_step_value"] = FusedPolicyStep(
                trainer(shape, "value", dev), rb, shape["B"], low, high, online=True)
            trs = transitions(cfg, 1000)
        else:
            trs = [None]
        for v in loops.values():
            host_steps(lambda i: v.step(trs[i % len(trs)]), args.warmup)

        def run(k, rep):
            us, last_loss[k] = host_steps(lambda i: loops[k].step(trs[i % len(trs)]),
                                          args.steps, rep * args.steps)
            return us

        per_update.update(alternate(loops, args.reps, run))

        # ac_value_rows_kernel alone, on the workspace of the "value" trainer
        t = loops[f"{sname}_train_batch_value"].t
        pins = Pins(dev)
        a, _ = t._value_args(b, t._ws, pins)
        desc, lib, cs = t.value_network.arena.desc(), _lib.lib(), _lib.cur_stream()
        ws = t._ws["value"].c

        def value_step():
            _lib.check(lib.rb200_ac_value_step(desc, a, ws, cs), "rb200_ac_value_step")

        kernel_us[sname] = [launch_us(value_step, args.launches) for _ in range(3)]
        del loops
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    med = {k: v["median"] for k, v in per_update.items()}
    res = {
        "what": ("per update: SACTrainer.train_batch without a value network, with one, and with "
                 "one plus CRR; the captured FusedPolicyStep step with a value network; "
                 "ac_value_rows_kernel alone"),
        "card": info,
        "shapes": SHAPES,
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed synchronised "
                   f"updates per variant after {args.warmup} warm-up updates; the captured step "
                   f"adds one transition to a 2^16 prioritized buffer each; the value kernel "
                   f"with the arguments SACTrainer._value_step builds: CUDA events over "
                   f"{args.launches} back-to-back launches after 10 warm-up launches, 3 "
                   f"repetitions"),
        "per_update_us": per_update,
        "value_vs_no_value_frac_median": {
            s: med[f"{s}_train_batch_value"] / med[f"{s}_train_batch_no_value"] - 1
            for s in SHAPES},
        "crr_vs_value_frac_median": {
            s: med[f"{s}_train_batch_crr"] / med[f"{s}_train_batch_value"] - 1 for s in SHAPES},
        "ac_value_rows_kernel_us": {s: dict(median=statistics.median(v), all=v)
                                    for s, v in kernel_us.items()},
        "last_loss": last_loss,
        "timestamp": time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime()),
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
