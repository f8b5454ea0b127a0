"""Time BehavioralCloningTrainer.train_batch against the same update written in eager torch, at
the size of a BCQ imitator for config-2 shapes (B 4096, FullyConnectedDQN 128-256-128-16 relu,
random masks, Adam lr 1e-3).

In one process, alternating the two variants:
  * `fused`: BehavioralCloningTrainer.train_batch (fused forward, rb200_bc_xent_head, fused
    backward and weight gradient, FusedAdam);
  * `eager`: nn.Sequential + masked logits + F.cross_entropy + backward + torch.optim.Adam, on
    the same GPU from the same initial weights and data;
and rb200_bc_xent_head alone with CUDA events.  The card's name, power limit and maximum SM
clock are read in the same run.

    python profiles/time_bc.py --out DIR [--reps 11] [--steps 200]

Writes DIR/time_bc.json and prints the same JSON.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.time_bcq import card_info, time_launches  # noqa: E402

B, S, A, SIZES, LR = 4096, 128, 16, [256, 128], 1e-3


def make_data(dev, n_batches=8):
    import torch

    g = torch.Generator().manual_seed(0)
    out = []
    for _ in range(n_batches):
        y = torch.randint(A, (B,), generator=g)
        mask = (torch.rand(B, A, generator=g) > 0.3).float()
        mask[torch.arange(B), y] = 1.0
        out.append(dict(state=torch.randn(B, S, generator=g).to(dev),
                        action=torch.nn.functional.one_hot(y, A).float().to(dev),
                        possible_actions_mask=mask.to(dev)))
    return out


def build(dev):
    import torch

    from reagent_b200.models import FullyConnectedDQN
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import BehavioralCloningTrainer

    torch.manual_seed(0)
    fused = BehavioralCloningTrainer(FullyConnectedDQN(S, A, SIZES, ["relu"] * len(SIZES)),
                                     optimizer=Optimizer__Union.default(lr=LR)).to(dev)
    layers = []
    dims = [S] + SIZES + [A]
    for i in range(len(dims) - 1):
        lin = torch.nn.Linear(dims[i], dims[i + 1])
        with torch.no_grad():
            lin.weight.copy_(fused.bc_net.fc.dnn[i][0].weight)
            lin.bias.copy_(fused.bc_net.fc.dnn[i][0].bias)
        layers.append(lin)
        if i < len(dims) - 2:
            layers.append(torch.nn.ReLU())
    eager = torch.nn.Sequential(*layers).to(dev)
    return fused, eager, torch.optim.Adam(eager.parameters(), lr=LR)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for time_bc.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=500)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F

    from reagent_b200 import _lib
    from reagent_b200.core import types as rlt

    if not torch.cuda.is_available():
        raise SystemExit("time_bc.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card_info()
    data = make_data(dev)
    batches = [rlt.BehavioralCloningModelInput(rlt.FeatureData(d["state"]), d["action"],
                                               d["possible_actions_mask"]) for d in data]
    fused, eager, opt = build(dev)

    def fused_step(i):
        return fused.train_batch(batches[i % len(batches)], i)

    def eager_step(i):
        d = data[i % len(data)]
        logits = eager(d["state"]) + (-1e10) * (1 - d["possible_actions_mask"])
        loss = F.cross_entropy(logits, d["action"].argmax(dim=1))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return loss.detach()

    variants = {"fused": fused_step, "eager": eager_step}
    # same weights, same first batch: the first losses agree
    first = {k: float(fn(0)) for k, fn in variants.items()}

    def run(fn, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(steps):
            loss = fn(i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps, float(loss)

    for fn in variants.values():
        run(fn, args.warmup)
    per_update = {k: [] for k in variants}
    last_loss = {}
    for rep in range(args.reps):
        order = list(variants) if rep % 2 == 0 else list(variants)[::-1]
        for k in order:
            dt, last_loss[k] = run(variants[k], args.steps)
            per_update[k].append(dt * 1e6)

    # the loss head alone, on the fused trainer's workspace
    ws = fused._ws
    d = data[0]
    a = _lib.BcXentArgsT()
    a.batch, a.num_actions = B, A
    a.logits, a.labels = ws["scores"].data_ptr(), d["action"].data_ptr()
    a.mask, a.dz = d["possible_actions_mask"].data_ptr(), ws["net"].dz[-1].data_ptr()
    a.loss_partials, a.loss = ws["loss_partials"].data_ptr(), ws["loss"].data_ptr()
    a.tile_counter = ws["counter"].data_ptr()
    lib, st = _lib.lib(), _lib.cur_stream()

    def head():
        _lib.check(lib.rb200_bc_xent_head(a, st), "rb200_bc_xent_head")

    head_us = [time_launches(head, args.launches) for _ in range(3)]

    med = {k: statistics.median(v) for k, v in per_update.items()}
    res = {
        "what": "BehavioralCloningTrainer.train_batch vs the same update in eager torch, per update",
        "card": info,
        "config": dict(B=B, S=S, A=A, sizes=SIZES, acts="relu", lr=LR, mask_keep=0.7),
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps, cycling over "
                   f"{len(data)} batches; head: CUDA events over {args.launches} back-to-back "
                   f"launches, 3 repetitions"),
        "per_update_us": {k: dict(median=med[k], min=min(v), max=max(v), all=v)
                          for k, v in per_update.items()},
        "speedup_median": med["eager"] / med["fused"],
        "bc_xent_head_us": dict(median=statistics.median(head_us), all=head_us),
        "first_loss": first,
        "last_loss": last_loss,
    }
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_bc.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
