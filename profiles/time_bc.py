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

Writes DIR/time_bc_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, card_info, cuda_device, host_steps,  # noqa: E402
                             launch_us, write_result)

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
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=500)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    import torch.nn.functional as F

    from reagent_b200 import _lib
    from reagent_b200.core import types as rlt

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

    for fn in variants.values():
        host_steps(fn, args.warmup)
    last_loss = {}

    def run(k, rep):
        us, last_loss[k] = host_steps(variants[k], args.steps)
        return us

    per_update = alternate(variants, args.reps, run)

    # the loss head alone, on the fused trainer's workspace
    d = data[0]
    a = fused._xent_args(fused._ws, d["action"], d["possible_actions_mask"])
    lib, st = _lib.lib(), _lib.cur_stream()

    def head():
        _lib.check(lib.rb200_bc_xent_head(a, st), "rb200_bc_xent_head")

    head_us = [launch_us(head, args.launches) for _ in range(3)]

    med = {k: v["median"] for k, v in per_update.items()}
    res = {
        "what": "BehavioralCloningTrainer.train_batch vs the same update in eager torch, per update",
        "card": info,
        "config": dict(B=B, S=S, A=A, sizes=SIZES, acts="relu", lr=LR, mask_keep=0.7),
        "method": (f"{args.reps} alternating repetitions of {args.steps} host-timed steps "
                   f"(synchronised) per variant after {args.warmup} warm-up steps, cycling over "
                   f"{len(data)} batches; head, with the arguments "
                   f"BehavioralCloningTrainer._step builds: CUDA events over {args.launches} "
                   f"back-to-back launches after 10 warm-up launches, 3 repetitions"),
        "per_update_us": per_update,
        "speedup_median": med["eager"] / med["fused"],
        "bc_xent_head_us": dict(median=statistics.median(head_us), all=head_us),
        "first_loss": first,
        "last_loss": last_loss,
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
