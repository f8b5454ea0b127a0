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

Writes DIR/time_sac_value.json and prints the same JSON.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from time_per import card_info, time_launches, time_steps, transitions  # noqa: E402

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
    ap.add_argument("--out", required=True, help="directory for time_sac_value.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    import random

    import numpy as np
    import torch

    import bench
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedPolicyStep
    from reagent_b200.training.workspace import Pins

    if not torch.cuda.is_available():
        raise SystemExit("time_sac_value.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
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
            time_steps(v, trs, args.warmup, 0)
        for k in loops:
            per_update[k] = []
        for rep in range(args.reps):
            order = list(loops) if rep % 2 == 0 else list(loops)[::-1]
            for k in order:
                dt, last_loss[k] = time_steps(loops[k], trs, args.steps, rep * args.steps)
                per_update[k].append(dt * 1e6)

        # ac_value_rows_kernel alone, on the workspace of the "value" trainer
        t = loops[f"{sname}_train_batch_value"].t
        pins = Pins(dev)
        a, _ = t._base_args(b, t._ws, pins)
        a.loss = t._ws["value_loss"].data_ptr()
        a.min_q_out = t._ws["min_q"].data_ptr()
        a.log_prob_out = t._ws["log_prob"].data_ptr()
        a.alpha = t._alpha_dev.data_ptr()
        a.logged_action_uniform_prior = 1
        desc, lib, cs = t.value_network.arena.desc(), _lib.lib(), _lib.cur_stream()
        ws = t._ws["value"].c

        def value_step():
            _lib.check(lib.rb200_ac_value_step(desc, a, ws, cs), "rb200_ac_value_step")

        kernel_us[sname] = [time_launches(value_step, args.launches) for _ in range(3)]
        del loops
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    med = {k: statistics.median(v) for k, v in per_update.items()}
    res = {
        "what": ("per update: SACTrainer.train_batch without a value network, with one, and with "
                 "one plus CRR; the captured FusedPolicyStep step with a value network; "
                 "ac_value_rows_kernel alone"),
        "card": info,
        "shapes": SHAPES,
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed synchronised "
                   f"updates per variant after {args.warmup} warm-up updates; the captured step "
                   f"adds one transition to a 2^16 prioritized buffer each; the value kernel: "
                   f"CUDA events over {args.launches} back-to-back launches, 3 repetitions"),
        "per_update_us": {k: dict(median=med[k], min=min(v), max=max(v), all=v)
                          for k, v in per_update.items()},
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
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_sac_value.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
