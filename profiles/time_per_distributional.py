"""Cost of prioritized experience replay for the distributional trainers
(FusedDqnStep(per=...) with QRDQNTrainer and C51Trainer).

Shapes: config 3 for QR-DQN (S 128, A 32, N 200, B 4096, replay capacity 2^20, q-network
128-256-128-(A*N) relu, double-Q) and the same trunk, A and B for C51 with N 51.  PER adds the
importance-weight kernel before the update, the weighted head instantiation, and the priority
write-back from the head's per-row losses (rb200_per_priority_update_rows, the ordered batched
SumTree.set) after it.  This script times, in one process:
  * FusedDqnStep(rng="device", online=True).step() per update with and without `per`, for both
    trainers, alternating the four variants;
  * the two priority write-backs alone at n = 4096 on a 2^20-leaf tree (TD-error priorities as
    DQN uses them, row-loss priorities as the distributional heads use them), with CUDA events
    over many launches;
and records the card's name, power limit and maximum SM clock read in the same run.

    python profiles/time_per_distributional.py --out DIR [--reps 11] [--steps 200]

Writes DIR/time_per_distributional.json and prints the same JSON.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from time_per import CAPACITY, card_info, time_launches, time_steps, transitions  # noqa: E402

C51_N, C51_QMIN, C51_QMAX = 51, -10.0, 10.0


def build_c51(cfg, dev, seed=0):
    import torch

    import bench
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import CategoricalDQN, FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import C51Trainer

    torch.manual_seed(seed)
    S, A, N = cfg["S"], cfg["A"], cfg["N"]
    q = CategoricalDQN(FullyConnectedDQN(S, A, cfg["sizes"], bench.ACTS, num_atoms=N),
                       qmin=C51_QMIN, qmax=C51_QMAX, num_atoms=N)
    qt = q.get_target_network()
    rl = RLParameters(gamma=bench.GAMMA, target_update_rate=bench.TAU)
    return C51Trainer(q.to(dev), qt.to(dev), actions=[str(i) for i in range(A)], rl=rl,
                      double_q_learning=True, minibatch_size=cfg["B"], num_atoms=N,
                      qmin=C51_QMIN, qmax=C51_QMAX,
                      optimizer=Optimizer__Union.default(lr=bench.LR)).to(dev)


def build(kind, cfg, dev, per):
    import bench
    from reagent_b200.replay_memory import PrioritizedReplayBuffer
    from reagent_b200.training.fused_step import FusedDqnStep

    rb = PrioritizedReplayBuffer(stack_size=1, replay_capacity=CAPACITY, batch_size=cfg["B"],
                                 device=dev)
    rb.add_batch(**bench.synth_stream(CAPACITY, 0, cfg))
    t = bench.build_trainer(cfg, dev, seed=0) if kind == "qrdqn" else build_c51(cfg, dev)
    return FusedDqnStep(t, rb, cfg["B"], rng="device", online=True, per=per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for time_per_distributional.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from reagent_b200 import _lib
    from reagent_b200.replay_memory import PrioritizedUpdate

    if not torch.cuda.is_available():
        raise SystemExit("time_per_distributional.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfgs = {"qrdqn": dict(bench.CONFIGS[3]), "c51": dict(bench.CONFIGS[3], N=C51_N)}
    info = card_info()
    per = PrioritizedUpdate(alpha=0.6, beta0=0.4, beta_updates=100_000, eps=1e-6)
    variants = {}
    for kind, cfg in cfgs.items():
        variants[f"{kind}_plain"] = build(kind, cfg, dev, None)
        variants[f"{kind}_per"] = build(kind, cfg, dev, per)
    trs = transitions(cfgs["qrdqn"], 1000)
    for fused in variants.values():
        time_steps(fused, trs, args.warmup, 0)
    per_update = {k: [] for k in variants}
    last_loss = {}
    for rep in range(args.reps):
        order = list(variants) if rep % 2 == 0 else list(variants)[::-1]
        for k in order:
            dt, last_loss[k] = time_steps(variants[k], trs, args.steps, rep * args.steps)
            per_update[k].append(dt * 1e6)
    for fused in variants.values():
        fused.dr.raise_if_failed()

    # the two write-backs alone: n = 4096 sets on a 2^20-leaf tree
    B = cfgs["qrdqn"]["B"]
    depth = 20
    rng = np.random.RandomState(0)
    tree = torch.from_numpy(rng.uniform(0.1, 10.0, (1 << (depth + 1)) - 1)).to(dev)
    idx = torch.from_numpy(rng.randint(0, CAPACITY, B).astype(np.int64)).to(dev)
    td = torch.from_numpy(rng.randn(B).astype(np.float32)).to(dev)
    qs = torch.from_numpy(rng.randn(B).astype(np.float32)).to(dev)
    rows = torch.from_numpy(rng.uniform(0.0, 4e4, B).astype(np.float32)).to(dev)
    p = torch.empty(B, dtype=torch.float64, device=dev)
    mx = torch.zeros(1, dtype=torch.float64, device=dev)
    st = torch.zeros(2, dtype=torch.int32, device=dev)
    lib, stream = _lib.lib(), _lib.cur_stream()

    def td_update():
        _lib.check(lib.rb200_per_priority_update(
            tree.data_ptr(), depth, idx.data_ptr(), td.data_ptr(), qs.data_ptr(), B, per.alpha,
            per.eps, p.data_ptr(), mx.data_ptr(), st.data_ptr(), stream))

    def rows_update():
        _lib.check(lib.rb200_per_priority_update_rows(
            tree.data_ptr(), depth, idx.data_ptr(), rows.data_ptr(), B, 200.0 * 200.0, per.alpha,
            per.eps, p.data_ptr(), mx.data_ptr(), st.data_ptr(), stream))

    kern = {}
    for rep in range(3):
        for name, fn in (("td_error_priority_update", td_update),
                         ("row_loss_priority_update", rows_update)):
            kern.setdefault(name, []).append(time_launches(fn, args.launches))
    torch.cuda.synchronize()
    assert int(st[0]) == 0

    med = {k: statistics.median(v) for k, v in per_update.items()}
    kmed = {k: statistics.median(v) for k, v in kern.items()}
    res = {
        "what": ("FusedDqnStep(rng='device', online=True).step() per update for QRDQNTrainer "
                 "(config 3) and C51Trainer (config-3 trunk, A and B; N 51), with and without "
                 "per; the TD-error and row-loss priority write-backs alone"),
        "card": info,
        "config": {k: dict(B=c["B"], S=c["S"], A=c["A"], N=c["N"], sizes=c["sizes"],
                           replay_capacity=CAPACITY) for k, c in cfgs.items()},
        "per": dict(alpha=per.alpha, beta0=per.beta0, beta_updates=per.beta_updates, eps=per.eps),
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps; write-backs: "
                   f"CUDA events over {args.launches} back-to-back launches, 3 repetitions, "
                   f"n = {B} sets on a 2^{depth}-leaf tree"),
        "per_update_us": {k: dict(median=med[k], min=min(v), max=max(v), all=v)
                          for k, v in per_update.items()},
        "per_overhead_us_median": {k: med[f"{k}_per"] - med[f"{k}_plain"] for k in cfgs},
        "per_overhead_frac_median": {k: med[f"{k}_per"] / med[f"{k}_plain"] - 1 for k in cfgs},
        "priority_update_us": {k: dict(median=kmed[k], all=v) for k, v in kern.items()},
        "last_loss": last_loss,
    }
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_per_distributional.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
