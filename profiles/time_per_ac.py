"""Cost of the captured online step and of prioritized replay for SACTrainer and TD3Trainer
(FusedPolicyStep).

Shapes: the per-GPU rows of configs 4 and 5 (SAC: S 256, A 32; TD3: S 512, A 64, delayed policy
update 2; both B 2048, twin critics, [256, 256] relu networks), replay capacity 2^20.  This
script times, in one process, alternating the variants of each trainer:
  * eager: the loop bench.py times end to end for these configs -- Python `random` draws on the
    host, a host->device copy of the query values, sample_policy_network_batch and train_batch
    launched eagerly (no transition added);
  * captured: FusedPolicyStep(rng="device", online=True).step(transition) -- add one transition,
    draw on the device and train, one CUDA graph replay;
  * captured_per: the same with per=PrioritizedUpdate(): importance weights, weighted critics and
    the twin-critic priority write-back inside the graph;
  * the priority write-back alone (rb200_per_priority_update_rows on the critics' TD errors) at
    n = 2048 on a 2^20-leaf tree, with CUDA events over many launches;
and records the card's name, power limit and maximum SM clock read in the same run.

    python profiles/time_per_ac.py --out DIR [--reps 11] [--steps 200]

Writes DIR/time_per_ac_<card>_<limit>w.json and prints the same JSON.
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

B = 2048
CAPACITY = 1 << 20


class EagerLoop:
    """Host draw -> pinned -> H2D of the query values -> sample kernel -> train_batch."""

    def __init__(self, trainer, rb, low, high):
        self.t, self.rb, self.low, self.high = trainer, rb, low, high
        self.i = 0

    def step(self, transition=None):
        import numpy as np
        import torch

        q, pos, idxs = self.rb.host_queries(B)
        kw = dict(query_dev=torch.from_numpy(np.ascontiguousarray(q)).pin_memory().to(
            self.rb._dev(), non_blocking=True))
        if pos:
            kw["overrides"] = (pos, idxs)
        batch = self.rb.sample_policy_network_batch(B, self.low, self.high, **kw)
        closs, _ = self.t.train_batch(batch, self.i)
        self.i += 1
        return closs


def build(cfg, dev, stream, variant, per):
    import numpy as np

    import bench
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedPolicyStep

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAPACITY, batch_size=B, device=dev)
    rb.add_batch(**stream)
    t = bench.build_trainer(cfg, dev, seed=0)
    low, high = -np.ones(cfg["A"], np.float32), np.ones(cfg["A"], np.float32)
    if variant == "eager":
        return EagerLoop(t, rb, low, high)
    return FusedPolicyStep(t, rb, B, low, high, online=True,
                           per=per if variant == "captured_per" else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    import random

    import numpy as np
    import torch

    import bench
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedUpdate

    random.seed(1234)
    cfgs = {"sac": dict(bench.CONFIGS[4], B=B), "td3": dict(bench.CONFIGS[5], B=B)}
    info = card_info()
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=100_000, eps=1e-6)
    names = ("eager", "captured", "captured_per")
    per_update, last_loss = {}, {}
    for algo, cfg in cfgs.items():
        stream = bench.synth_stream(CAPACITY, 0, cfg)
        variants = {f"{algo}_{v}": build(cfg, dev, stream, v, per) for v in names}
        del stream
        trs = transitions(cfg, 1000)
        for v in variants.values():
            host_steps(lambda i: v.step(trs[i % len(trs)]), args.warmup)

        def run(k, rep):
            us, last_loss[k] = host_steps(lambda i: variants[k].step(trs[i % len(trs)]),
                                          args.steps, rep * args.steps)
            return us

        per_update.update(alternate(variants, args.reps, run))
        for k, v in variants.items():
            if hasattr(v, "dr"):
                v.dr.raise_if_failed()
        del variants
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    # the twin-critic priority write-back alone: n = 2048 sets on a 2^20-leaf tree
    depth = 20
    rng = np.random.RandomState(0)
    tree = torch.from_numpy(rng.uniform(0.1, 10.0, (1 << (depth + 1)) - 1)).to(dev)
    idx = torch.from_numpy(rng.randint(0, CAPACITY, B).astype(np.int64)).to(dev)
    td = torch.from_numpy(np.abs(rng.randn(B)).astype(np.float32)).to(dev)
    p = torch.empty(B, dtype=torch.float64, device=dev)
    mx = torch.zeros(1, dtype=torch.float64, device=dev)
    st = torch.zeros(2, dtype=torch.int32, device=dev)
    lib, cs = _lib.lib(), _lib.cur_stream()

    def write_back():
        _lib.check(lib.rb200_per_priority_update_rows(
            tree.data_ptr(), depth, idx.data_ptr(), td.data_ptr(), B, 1.0, per.alpha, per.eps,
            p.data_ptr(), mx.data_ptr(), st.data_ptr(), cs))

    wb = [launch_us(write_back, args.launches) for _ in range(3)]
    torch.cuda.synchronize()
    assert int(st[0]) == 0

    med = {k: v["median"] for k, v in per_update.items()}
    res = {
        "what": ("per update: the eager host-RNG loop, FusedPolicyStep(rng='device', "
                 "online=True).step() without and with per, for SACTrainer (config-4 per-GPU "
                 "shapes) and TD3Trainer (config-5 per-GPU shapes); the twin-critic priority "
                 "write-back alone"),
        "card": info,
        "config": {k: dict(B=B, S=c["S"], A=c["A"], sizes=c["sizes"], replay_capacity=CAPACITY,
                           twin_critics=True) for k, c in cfgs.items()},
        "per": dict(alpha=per.alpha, beta0=per.beta0, beta_updates=per.beta_updates, eps=per.eps),
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps; the eager "
                   f"loop adds no transition, the captured steps add one each; write-back: CUDA "
                   f"events over {args.launches} back-to-back launches after 10 warm-up "
                   f"launches, 3 repetitions, n = {B} sets on a 2^{depth}-leaf tree"),
        "per_update_us": per_update,
        "captured_vs_eager_frac_median": {a: med[f"{a}_captured"] / med[f"{a}_eager"] - 1
                                          for a in cfgs},
        "per_overhead_us_median": {a: med[f"{a}_captured_per"] - med[f"{a}_captured"]
                                   for a in cfgs},
        "priority_write_back_us": dict(median=statistics.median(wb), all=wb),
        "last_loss": last_loss,
        "timestamp": time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime()),
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
