"""Time MDNRNNTrainer.train_batch against the same update written in eager torch: nn.LSTM
(cuDNN), nn.Linear, the reference's loss formulas (gmm_loss, binary_cross_entropy_with_logits,
mse_loss; loss = gmm / (S + 2) + bce + mse) and torch.optim.Adam(foreach=True).

Shapes (T, B, S, A, H, L, G):
  * cartpole_features: 1, 1024, 4, 2, 50, 2, 1   (configs/world_model/cartpole_features.yaml)
  * cem_cartpole:      1, 1024, 4, 2, 100, 2, 1  (the mdnrnn block of cem_cartpole_offline.yaml)
  * defaults_t1:       1, 1024, 4, 2, 64, 2, 5   (MDNRNNTrainerParameters() defaults)
  * defaults_t16:      16, 1024, 4, 2, 64, 2, 5

In one process per shape, alternating the two variants:
  * `fused`: MDNRNNTrainer.train_batch (rb200_mdnrnn_forward, _backward, _wgrad, FusedAdam);
  * `eager`: the update above, from the same initial weights and data;
and rb200_mdnrnn_forward alone (forward + losses + dL/d(gmm_outs)) with CUDA events.  The
card's name, power limit and maximum SM clock are read in the same run.

    python profiles/time_mdnrnn.py --out DIR [--reps 7] [--steps 100]

Writes DIR/time_mdnrnn_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import (alternate, card_info, cuda_device, host_steps,  # noqa: E402
                             launch_us, write_result)

SHAPES = {
    "cartpole_features": dict(T=1, B=1024, S=4, A=2, H=50, L=2, G=1),
    "cem_cartpole": dict(T=1, B=1024, S=4, A=2, H=100, L=2, G=1),
    "defaults_t1": dict(T=1, B=1024, S=4, A=2, H=64, L=2, G=5),
    "defaults_t16": dict(T=16, B=1024, S=4, A=2, H=64, L=2, G=5),
}
LR = 1e-3


def make_data(dev, T, B, S, A, n_batches=4):
    import torch

    g = torch.Generator().manual_seed(0)
    out = []
    for _ in range(n_batches):
        act = torch.nn.functional.one_hot(torch.randint(A, (T, B), generator=g), A).float()
        out.append(dict(state=torch.randn(T, B, S, generator=g).to(dev), action=act.to(dev),
                        next_state=torch.randn(T, B, S, generator=g).to(dev),
                        reward=torch.randn(T, B, generator=g).to(dev),
                        not_terminal=(torch.rand(T, B, generator=g) > 0.05).float().to(dev)))
    return out


def eager_loss(lstm, head, d, S, G):
    """The reference's MDNRNN.forward and get_loss, in eager torch."""
    import torch
    import torch.nn.functional as F

    T, B = d["state"].shape[:2]
    h, _ = lstm(torch.cat([d["action"], d["state"]], dim=-1))
    y = head(h)
    GS = G * S
    mus = y[:, :, :GS].view(T, B, G, S)
    sigmas = torch.exp(y[:, :, GS:2 * GS].view(T, B, G, S))
    logpi = F.log_softmax(y[:, :, 2 * GS:2 * GS + G], dim=-1)
    x = d["next_state"].unsqueeze(-2)
    lp = -((x - mus) ** 2) / (2 * sigmas ** 2) - sigmas.log() - math.log(math.sqrt(2 * math.pi))
    z = logpi + lp.sum(dim=-1)
    m = z.max(dim=-1, keepdim=True)[0]
    gmm = -(m.squeeze(-1) + torch.log(torch.exp(z - m).sum(dim=-1))).mean()
    bce = F.binary_cross_entropy_with_logits(y[:, :, -1], d["not_terminal"])
    mse = F.mse_loss(y[:, :, -2], d["reward"])
    return gmm / (S + 2) + bce + mse


def time_shape(name, cfg, args, dev):
    import torch

    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import MDNRNNTrainerParameters
    from reagent_b200.models import MemoryNetwork
    from reagent_b200.training import MDNRNNTrainer

    T, B, S, A, H, L, G = (cfg[k] for k in ("T", "B", "S", "A", "H", "L", "G"))
    data = make_data(dev, T, B, S, A)
    batches = [rlt.MemoryNetworkInput(
        state=rlt.FeatureData(d["state"]), next_state=rlt.FeatureData(d["next_state"]),
        action=rlt.FeatureData(d["action"]), reward=d["reward"], not_terminal=d["not_terminal"],
        time_diff=None, step=None) for d in data]
    torch.manual_seed(0)
    net = MemoryNetwork(S, A, H, L, G)
    lstm, head = torch.nn.LSTM(S + A, H, L).to(dev), torch.nn.Linear(H, (2 * S + 1) * G + 2).to(dev)
    with torch.no_grad():
        for p, q in zip(list(lstm.parameters()) + list(head.parameters()), net.mdnrnn.parameters()):
            p.copy_(q)
    fused = MDNRNNTrainer(net.to(dev), MDNRNNTrainerParameters(
        hidden_size=H, num_hidden_layers=L, num_gaussians=G, action_dim=A, learning_rate=LR))
    params = list(lstm.parameters()) + list(head.parameters())
    opt = torch.optim.Adam(params, lr=LR, foreach=True)

    def fused_step(i):
        return fused.train_batch(batches[i % len(batches)], i)[3]

    def eager_step(i):
        loss = eager_loss(lstm, head, data[i % len(data)], S, G)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return loss.detach()

    variants = {"fused": fused_step, "eager": eager_step}
    first = {k: float(fn(0)) for k, fn in variants.items()}
    for fn in variants.values():
        host_steps(fn, args.warmup)
    last_loss = {}

    def run(k, rep):
        us, last_loss[k] = host_steps(variants[k], args.steps)
        return us

    per_update = alternate(variants, args.reps, run)

    # forward + losses + dL/d(gmm_outs) alone, with the arguments MDNRNNTrainer._step builds
    from reagent_b200 import _lib

    b, p, ws = data[0], fused.params, fused._ws
    a = net.mdnrnn.args(T, B)
    a.state, a.action = b["state"].data_ptr(), b["action"].data_ptr()
    a.next_state, a.reward = b["next_state"].data_ptr(), b["reward"].data_ptr()
    a.not_terminal = b["not_terminal"].data_ptr()
    a.next_state_weight, a.not_terminal_weight = p.next_state_loss_weight, p.not_terminal_loss_weight
    a.reward_weight, a.gmm_divisor, a.fit_only_one_next_step = p.reward_loss_weight, S + 2.0, 0
    for f in ("out", "hs", "cs", "xin", "acts", "dgates", "dy", "loss"):
        setattr(a, f, getattr(ws, f).data_ptr())
    a.loss_partials, a.tile_counter = ws.loss_partials.data_ptr(), ws.counter.data_ptr()
    lib, st = _lib.lib(), _lib.cur_stream()

    def fwd():
        _lib.check(lib.rb200_mdnrnn_forward(a, st), "rb200_mdnrnn_forward")

    fwd_us = [launch_us(fwd, args.launches) for _ in range(3)]
    med = {k: v["median"] for k, v in per_update.items()}
    return {"config": dict(cfg, lr=LR), "per_update_us": per_update,
            "speedup_median": med["eager"] / med["fused"],
            "forward_loss_kernel_us": dict(median=statistics.median(fwd_us), all=fwd_us),
            "first_loss": first, "last_loss": last_loss}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    info = card_info()
    res = {
        "what": "MDNRNNTrainer.train_batch vs the same update in eager torch (cuDNN LSTM), "
                "per update",
        "card": info,
        "method": (f"per shape, {args.reps} alternating repetitions of {args.steps} host-timed "
                   f"steps (synchronised) per variant after {args.warmup} warm-up steps, cycling "
                   "over 4 batches; rb200_mdnrnn_forward with the arguments MDNRNNTrainer._step "
                   f"builds: CUDA events over {args.launches} back-to-back launches after 10 "
                   "warm-up launches, 3 repetitions"),
        "shapes": {name: time_shape(name, cfg, args, dev) for name, cfg in SHAPES.items()},
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
