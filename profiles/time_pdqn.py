"""What the fused tiled next-action forward (rb200_mlp_forward_tiled) saves in the max-Q update
of ParametricDQNTrainer.  One process; records the card's name, power limit and maximum SM
clock read in the same run.

Two variants of the same double-Q, max-Q `train_batch` (with the reward network):
  fused         the trainer as shipped: one launch scores both networks on every
                (next state, possible next action) pair, the tiled input built in shared memory;
  materialised  the path it replaced, rebuilt here: next_state.repeat_interleave(M) + torch.cat
                with the possible next actions, then one rb200_mlp_forward per network.
Both give bit-identical results.  For each variant a CUDA graph of --iters back-to-back
`train_batch` calls is captured and one replay is timed with CUDA events; the next-state
forward alone (the part that differs) is timed the same way.  The variants run alternately,
--reps times each, and the median is reported.

Shapes: the CartPole configuration (S 4, A 2, [128, 64] leaky_relu, B 1024) and
S 128 / A 16 / B 4096 / [256, 128] relu, one-hot actions with the identity tiling.

    python profiles/time_pdqn.py --out DIR [--reps 11] [--iters 50]

Writes DIR/time_pdqn.json and prints the same JSON.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.time_k2 import card_info  # noqa: E402

SHAPES = {
    "cartpole": dict(S=4, A=2, B=1024, sizes=[128, 64], act="leaky_relu"),
    "s128_a16_b4096": dict(S=128, A=16, B=4096, sizes=[256, 128], act="relu"),
}


def materialised(arenas, state, actions, M, outs):
    """The replaced path: the tiled input in HBM, then one forward per network."""
    import torch

    from reagent_b200.models.arena import run_mlp

    x = torch.cat((state.repeat_interleave(M, dim=0), actions), dim=1).contiguous()
    for a, o in zip(arenas, outs):
        run_mlp(a.desc(), x, o)


def build(shape):
    import torch

    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import RLParameters
    from reagent_b200.models import FullyConnectedCritic
    from reagent_b200.optimizer import Optimizer__Union
    from reagent_b200.training import ParametricDQNTrainer

    S, A, B = shape["S"], shape["A"], shape["B"]
    acts = [shape["act"]] * len(shape["sizes"])
    torch.manual_seed(0)
    q = FullyConnectedCritic(S, A, shape["sizes"], acts).cuda()
    rn = FullyConnectedCritic(S, A, shape["sizes"], acts).cuda()
    t = ParametricDQNTrainer(q, q.get_target_network(), rn,
                             rl=RLParameters(gamma=0.99, target_update_rate=0.1),
                             double_q_learning=True,
                             optimizer=Optimizer__Union(AdamW={"lr": 1e-3, "amsgrad": True})).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randint(A, (B,), device="cuda", generator=g)
    eye = torch.eye(A, device="cuda").repeat(B, 1)
    batch = rlt.ParametricDqnInput(
        state=rlt.FeatureData(torch.randn(B, S, device="cuda", generator=g)),
        next_state=rlt.FeatureData(torch.randn(B, S, device="cuda", generator=g)),
        reward=torch.randn(B, 1, device="cuda", generator=g), time_diff=None, step=None,
        not_terminal=torch.ones(B, 1, device="cuda"),
        action=rlt.FeatureData(torch.nn.functional.one_hot(a, A).float()),
        next_action=rlt.FeatureData(torch.nn.functional.one_hot(a, A).float()),
        possible_actions=rlt.FeatureData(eye), possible_actions_mask=torch.ones(B, A, device="cuda"),
        possible_next_actions=rlt.FeatureData(eye),
        possible_next_actions_mask=torch.ones(B, A, device="cuda"), extras=rlt.ExtraData())
    return t, batch


def capture(fn, iters):
    import torch

    fn()  # warm-up: lazy allocations, module load, optimizer state
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(iters):
            fn()
    torch.cuda.synchronize()
    return g


def time_graph(g, iters):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters  # us per call


def variants(shape, iters):
    """{(variant, what): graph} for one shape; every graph keeps its own trainer alive."""
    import torch

    import reagent_b200.training.parametric_dqn_trainer as mod

    fused_fn = mod.run_mlp_tiled
    out, keep = {}, []
    for name, fwd in (("fused", fused_fn), ("materialised", materialised)):
        mod.run_mlp_tiled = fwd
        try:
            t, batch = build(shape)
            out[(name, "train_batch")] = capture(lambda: t.train_batch(batch), iters)
            B = batch.state.float_features.shape[0]
            M = batch.possible_next_actions.float_features.shape[0] // B
            ns = batch.next_state.float_features
            pna = batch.possible_next_actions.float_features
            outs = [torch.empty(B * M, 1, device="cuda") for _ in range(2)]
            arenas = [t.q_network_target.arena, t.q_network.arena]
            out[(name, "next_q_forward")] = capture(lambda: fwd(arenas, ns, pna, M, outs), iters)
            keep.append((t, batch, outs))
        finally:
            mod.run_mlp_tiled = fused_fn
    return out, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for time_pdqn.json")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch

    torch.cuda.set_device(0)
    result = {"card": card_info(), "reps": args.reps, "iters_per_graph": args.iters,
              "unit": "us per call, median [min, max] over reps", "shapes": {}}
    for sname, shape in SHAPES.items():
        graphs, keep = variants(shape, args.iters)
        times = {k: [] for k in graphs}
        for r in range(args.reps):
            order = sorted(graphs) if r % 2 == 0 else sorted(graphs, reverse=True)
            for k in order:
                times[k].append(time_graph(graphs[k], args.iters))
        res = {"shape": shape}
        for (variant, what), v in times.items():
            res.setdefault(what, {})[variant] = {"median": statistics.median(v), "min": min(v),
                                                 "max": max(v)}
        for what in ("train_batch", "next_q_forward"):
            r = res[what]
            r["materialised_over_fused"] = r["materialised"]["median"] / r["fused"]["median"]
        result["shapes"][sname] = res
        del graphs, keep
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_pdqn.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
