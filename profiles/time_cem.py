"""Time one CEM act() (CEMPolicy.act: a whole plan and reading its action) against the same plan
in eager torch, and the rollout kernel alone.

Configurations (the reference's configs/world_model/cem_*.yaml; seeded, untrained world models
of hidden 100, 2 layers, 1 gaussian):
  * cartpole:      discrete, K 1, S 4, A 2, H 10, P 100, terminal effective, gamma 1
  * linear_single: continuous in [-3, 3], K 1, S 3, A 2, H 4, P 100, 10 iterations, 15 elites
  * linear_many:   the same with K 2

In one process per configuration, alternating the variants:
  * `fused`: CEMPolicy.act (noise drawn on the GPU, one rb200_cem_rollout launch per CEM
    iteration, the action copied to the host);
  * `eager`: the same plan in eager torch on the same GPU, batched over the population (the
    zero-state LSTM step, mixture / normal / Bernoulli draws from the same kind of noise, the
    elite update in fp64, and the early-stop check on the host every iteration, as the
    reference does);
  * at cartpole, `reference_loop`: the reference's per-trajectory loop (one single-row world
    model forward per step with torch.distributions samplers and .item()) on the GPU.
rb200_cem_rollout alone: CUDA events around each launch of iteration 0 (the planner's state is
reset before each, outside the events).  The card's name, power limit and maximum SM clock are
read in the same run.

    python profiles/time_cem.py --out DIR [--reps 5] [--acts 20]

Writes DIR/time_cem_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import alternate, card_info, cuda_device, summary, write_result  # noqa: E402

CONFIGS = {
    "cartpole": dict(discrete=True, K=1, S=4, A=2, H=10, P=100, iters=10, E=15, terminal=True),
    "linear_single": dict(discrete=False, K=1, S=3, A=2, H=4, P=100, iters=10, E=15,
                          terminal=False),
    "linear_many": dict(discrete=False, K=2, S=3, A=2, H=4, P=100, iters=10, E=15,
                        terminal=False),
}
HIDDEN, LAYERS, G, GAMMA, BOUND = 100, 2, 1, 1.0, 3.0


def _weights(net):
    """(per layer (W_ih, b_ih, b_hh), W_gmm, b_gmm) of a MemoryNetwork."""
    ps = list(net.mdnrnn.parameters())
    layers = [(ps[4 * l], ps[4 * l + 2], ps[4 * l + 3]) for l in range(LAYERS)]
    return layers, ps[-2], ps[-1]


def _step(W, x):
    """One T = 1 world-model step from h = c = 0: the gmm head output."""
    import torch

    layers, wg, bg = W
    h = x
    for w_ih, b_ih, b_hh in layers:
        i, _, g, o = (b_hh + (h @ w_ih.T + b_ih)).chunk(4, dim=1)
        h = torch.sigmoid(o) * torch.tanh(torch.sigmoid(i) * torch.tanh(g))
    return h @ wg.T + bg


def eager_plan(models, cfg, state, noise, lo, hi, eps=0.001, alpha=0.25):
    """The plan of CEMPlannerNetwork in eager torch, batched over the population."""
    import torch
    import torch.nn.functional as F

    P, H, A, S, K = cfg["P"], cfg["H"], cfg["A"], cfg["S"], cfg["K"]
    GS, dev = G * S, state.device
    disc = torch.tensor([GAMMA ** j for j in range(H)], device=dev)
    mean, var = (hi + lo) / 2, (hi - lo) ** 2 / 16
    rows = torch.arange(P, device=dev)
    for it in range(1 if cfg["discrete"] else cfg["iters"]):
        if cfg["discrete"]:
            acts = F.one_hot(noise.action_idx.long(), A).float()
        else:
            cv = torch.minimum(torch.minimum(((mean - lo) / 2) ** 2, ((hi - mean) / 2) ** 2), var)
            sol = noise.truncnorm[it] * cv.sqrt() + mean
            acts = sol.view(P, H, A).float()
        midx = noise.model_idx[it].long()
        xs = state.expand(P, S)
        alive = torch.ones(P, dtype=torch.bool, device=dev)
        val = torch.zeros(P, dtype=torch.float64, device=dev)
        for j in range(H):
            x = torch.cat([acts[:, j], xs], dim=1)
            y = _step(models[0], x)
            for m in range(1, K):
                y = torch.where((midx == m)[:, None], _step(models[m], x), y)
            nz = noise.step[it, :, j]
            p = F.softmax(y[:, 2 * GS:2 * GS + G], dim=1)
            k = (nz[:, :1] * p.sum(1, keepdim=True) < p.cumsum(1)).int().argmax(1)
            mus, sig = y[:, :GS].view(P, G, S), y[:, GS:2 * GS].exp().view(P, G, S)
            ns = mus[rows, k] + sig[rows, k] * nz[:, 1:S + 1]
            val += torch.where(alive, (y[:, -2] * disc[j]).double(), 0.0)
            if cfg["terminal"]:
                alive = alive & (nz[:, S + 1] < torch.sigmoid(y[:, -1]))
            xs = torch.where(alive[:, None], ns, xs)
        if cfg["discrete"]:
            first = noise.action_idx[:, 0].long()
            cnt = torch.zeros(A, dtype=torch.float64, device=dev).index_add_(0, first, torch.ones_like(val))
            tally = torch.zeros(A, dtype=torch.float64, device=dev).index_add_(0, first, val)
            return torch.nan_to_num(tally / cnt, nan=-float("inf")).argmax().cpu()
        el = sol[val.topk(cfg["E"]).indices]
        mean = alpha * mean + (1 - alpha) * el.mean(0)
        var = alpha * var + (1 - alpha) * el.var(0, unbiased=False)
        if var.max().item() <= eps:
            break
    return (((mean[:A] - lo[:A]) / (hi[:A] - lo[:A])) * 2.0 - 1.0).cpu()


def reference_loop(models, cfg, state):
    """The reference's acc_rewards_of_all_solutions + discrete_planning, on the GPU."""
    import numpy as np
    import torch
    from torch.distributions import Bernoulli, Categorical, Normal

    P, H, A, S = cfg["P"], cfg["H"], cfg["A"], cfg["S"]
    GS = G * S
    seqs = np.random.randint(0, A, size=(P, H))
    acc = np.zeros(P)
    for i in range(P):
        W = models[np.random.randint(0, len(models))]
        st = state
        for j in range(H):
            a = torch.zeros(1, A, device=state.device)
            a[0, seqs[i, j]] = 1
            y = _step(W, torch.cat([a, st], dim=1))[0]
            logpi = torch.log_softmax(y[2 * GS:2 * GS + G], 0)
            k = Categorical(torch.exp(logpi)).sample().long().item()
            st = Normal(y[k * S:(k + 1) * S], y[GS + k * S:GS + (k + 1) * S].exp()).sample()[None]
            acc[i] += float(y[-2]) * (GAMMA ** j)
            if not Bernoulli(torch.sigmoid(y[-1])).sample().long().item():
                break
    cnt, tally = np.zeros(A), np.zeros(A)
    for f, v in zip(seqs[:, 0], acc):
        cnt[f] += 1
        tally[f] += v
    with np.errstate(invalid="ignore"):
        return int(np.nanargmax(tally / cnt))


def time_config(name, cfg, args, dev):
    import numpy as np
    import torch

    from reagent_b200 import _lib
    from reagent_b200.core import types as rlt
    from reagent_b200.model_managers import CEMPolicy
    from reagent_b200.models import CEMPlannerNetwork, MemoryNetwork

    torch.manual_seed(0)
    S, A = cfg["S"], cfg["A"]
    nets = [MemoryNetwork(S, A, HIDDEN, LAYERS, G).to(dev) for _ in range(cfg["K"])]
    bounds = np.full(A, BOUND)
    planner = CEMPlannerNetwork(
        nets, cfg["iters"], cfg["P"], 1, cfg["E"], cfg["H"], S, A, cfg["discrete"],
        cfg["terminal"], GAMMA, action_upper_bounds=None if cfg["discrete"] else bounds,
        action_lower_bounds=None if cfg["discrete"] else -bounds)
    policy = CEMPolicy(planner, cfg["discrete"])
    obs = rlt.FeatureData(torch.randn(1, S, device=dev))
    models = [_weights(n) for n in nets]
    lo = torch.full((cfg["H"] * A,), -BOUND, dtype=torch.float64, device=dev)
    hi = -lo
    noise = planner.new_noise(dev)

    def fused():
        return policy.act(obs)

    def eager():
        return eager_plan(models, cfg, obs.float_features, noise.fill_(), lo, hi)

    variants = {"fused": fused, "eager": eager}
    if name == "cartpole":
        variants["reference_loop"] = lambda: reference_loop(models, cfg, obs.float_features)
    for fn in variants.values():
        for _ in range(3):
            fn()

    def run(k, rep):
        n = 1 if k == "reference_loop" else args.acts
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            variants[k]()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n * 1e6

    per_act = alternate(variants, args.reps, run)
    p = planner.plan(obs)
    n_iters = int(p.n_iters.item())

    # rb200_cem_rollout alone: iteration 0, with the planner's state reset outside the events
    ws = planner._ws
    a = planner._args(ws, ws.noise.fill_(), None)
    a.iter = 0
    lib, st = _lib.lib(), _lib.cur_stream()
    kernel_us = []
    for _ in range(3):
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
               for _ in range(args.launches)]
        for e0, e1 in evs:
            ws.done.zero_()
            if not cfg["discrete"]:
                ws.mean.copy_(ws.mean0)
                ws.var.copy_(ws.var0)
            e0.record()
            _lib.check(lib.rb200_cem_rollout(a, st), "rb200_cem_rollout")
            e1.record()
        torch.cuda.synchronize()
        kernel_us.append(statistics.median(e0.elapsed_time(e1) * 1e3 for e0, e1 in evs))
    med = {k: v["median"] for k, v in per_act.items()}
    return {"config": dict(cfg, hidden=HIDDEN, layers=LAYERS, gaussians=G, gamma=GAMMA),
            "per_act_us": per_act,
            "speedup_median": {k: med[k] / med["fused"] for k in med if k != "fused"},
            "fused_iterations_run": n_iters,
            "rollout_kernel_us": summary(kernel_us)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--acts", type=int, default=20)
    ap.add_argument("--launches", type=int, default=100)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    info = card_info()
    res = {
        "what": "one CEMPolicy.act (a whole plan, action read on the host) vs the same plan in "
                "eager torch batched over the population, and rb200_cem_rollout alone",
        "card": info,
        "method": (f"per configuration, {args.reps} alternating repetitions of {args.acts} "
                   "host-timed acts (synchronised) per variant after 3 warm-up acts; the "
                   "reference-style loop: one act per repetition; rb200_cem_rollout: CUDA events "
                   f"around each of {args.launches} launches of iteration 0, median, 3 "
                   "repetitions"),
        "configs": {name: time_config(name, cfg, args, dev) for name, cfg in CONFIGS.items()},
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
