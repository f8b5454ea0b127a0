"""Time the world-model evaluators (FeatureImportanceEvaluator + FeatureSensitivityEvaluator)
against the reference's algorithm in eager torch on the same GPU.

Shapes (T, B, S, A, H, L, G):
  * cartpole_features: 1, 6000, 4, 2 discrete, 50, 2, 1  (test_world_model.py's test batch)
  * defaults_t16:      16, 1024, 4, 2 discrete, 64, 2, 5  (MDNRNNTrainerParameters() defaults)
  * wide:              1, 4096, 64, 4 continuous, 64, 2, 5

In one process per shape, alternating the two variants, host-clocked including the read-back:
  * `fused`: FeatureImportanceEvaluator.evaluate then FeatureSensitivityEvaluator.evaluate
    (rb200_mdnrnn_fill_values, one rb200_mdnrnn_eval launch over 1 + A + S variants, one over
    2 variants with the means, rb200_mdnrnn_sensitivity; one read-back each);
  * `eager`: the reference's loop -- per feature, clone the batch, set the feature, the loss of
    profiles/time_mdnrnn.eager_loss (cuDNN LSTM) and .item() -- plus the two forwards and the
    per-feature mean |delta mu| of the sensitivity, from the same weights and data;
and rb200_mdnrnn_eval of the importance variants alone with CUDA events.  The card's name, power
limit and maximum SM clock are read in the same run.

    python profiles/time_world_model_eval.py --out DIR [--reps 7] [--iters 20]

Writes DIR/time_world_model_eval_<card>_<limit>w.json and prints the same JSON.
"""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.timing import alternate, card_info, cuda_device, launch_us, write_result  # noqa: E402

SHAPES = {
    "cartpole_features": dict(T=1, B=6000, S=4, A=2, H=50, L=2, G=1, discrete=True),
    "defaults_t16": dict(T=16, B=1024, S=4, A=2, H=64, L=2, G=5, discrete=True),
    "wide": dict(T=1, B=4096, S=64, A=4, H=64, L=2, G=5, discrete=False),
}


def make_batch(dev, T, B, S, A, discrete):
    import torch

    g = torch.Generator().manual_seed(0)
    if discrete:
        act = torch.nn.functional.one_hot(torch.randint(A, (T, B), generator=g), A).float()
    else:
        act = torch.rand(T, B, A, generator=g) * 2 - 1
    return dict(state=torch.randn(T, B, S, generator=g).to(dev), action=act.to(dev),
                next_state=torch.randn(T, B, S, generator=g).to(dev),
                reward=torch.randn(T, B, generator=g).to(dev),
                not_terminal=(torch.rand(T, B, generator=g) > 0.05).float().to(dev))


def eager_evaluate(lstm, head, d, S, A, G, discrete, perm):
    """The reference's FeatureImportanceEvaluator and FeatureSensitivityEvaluator (every
    feature one column wide), with eager_loss as get_loss."""
    import torch

    from profiles.time_mdnrnn import eager_loss

    T, B = d["state"].shape[:2]
    with torch.no_grad():
        imp = torch.zeros(A + S)
        orig = eager_loss(lstm, head, d, S, G).item()
        for i in range(A):
            act = d["action"].reshape(T * B, A).clone()
            if discrete:
                v = torch.zeros(A, device=act.device)
                v[i] = 1
                act[:] = v
            else:
                act[:, i:i + 1] = act[:, i:i + 1].mean(dim=0)
            imp[i] = eager_loss(lstm, head, dict(d, action=act.reshape(T, B, A)), S, G).item() - orig
        for i in range(S):
            st = d["state"].reshape(T * B, S).clone()
            st[:, i:i + 1] = st[:, i:i + 1].mean(dim=0)
            imp[A + i] = eager_loss(lstm, head, dict(d, state=st.reshape(T, B, S)), S, G).item() - orig

        def mus(action):
            h, _ = lstm(torch.cat([action, d["state"]], dim=-1))
            return head(h)[:, :, :G * S].view(T, B, G, S)

        m0, m1 = mus(d["action"]), mus(d["action"][:, perm, :])
        sens = torch.zeros(S)
        for i in range(S):
            sens[i] = (m1[..., i:i + 1] - m0[..., i:i + 1]).abs().sum(dim=3).mean().item()
    return imp, sens


def time_shape(name, cfg, args, dev):
    import torch

    from reagent_b200.core import types as rlt
    from reagent_b200.core.parameters import MDNRNNTrainerParameters
    from reagent_b200.evaluation import FeatureImportanceEvaluator, FeatureSensitivityEvaluator
    from reagent_b200.models import MemoryNetwork
    from reagent_b200.training import MDNRNNTrainer

    T, B, S, A, H, L, G = (cfg[k] for k in "TBSAHLG")
    discrete = cfg["discrete"]
    torch.manual_seed(0)
    net = MemoryNetwork(S, A, H, L, G)
    lstm = torch.nn.LSTM(S + A, H, L).to(dev)
    head = torch.nn.Linear(H, (2 * S + 1) * G + 2).to(dev)
    with torch.no_grad():
        for p, q in zip(list(lstm.parameters()) + list(head.parameters()),
                        net.mdnrnn.parameters()):
            p.copy_(q)
    tr = MDNRNNTrainer(net.to(dev), MDNRNNTrainerParameters(
        hidden_size=H, num_hidden_layers=L, num_gaussians=G, action_dim=A))
    d = make_batch(dev, T, B, S, A, discrete)
    batch = rlt.MemoryNetworkInput(
        state=rlt.FeatureData(d["state"]), next_state=rlt.FeatureData(d["next_state"]),
        action=rlt.FeatureData(d["action"]), reward=d["reward"], not_terminal=d["not_terminal"],
        time_diff=None, step=None)
    imp = FeatureImportanceEvaluator(tr, discrete, S, A, list(range(A)), list(range(S)))
    sens = FeatureSensitivityEvaluator(tr, S, list(range(S)))
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1))
    perm_dev = perm.to(dev)

    def fused():
        return (imp.evaluate(batch)["feature_loss_increase"],
                sens.evaluate(batch, perm=perm)["feature_sensitivity"])

    def eager():
        return eager_evaluate(lstm, head, d, S, A, G, discrete, perm_dev)

    calls = {"fused": fused, "eager": eager}
    results = {}
    for k, fn in calls.items():
        for _ in range(args.warmup):
            results[k] = fn()

    def run(k, rep):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            calls[k]()
        return (time.perf_counter() - t0) / args.iters * 1e6

    per_eval = alternate(calls, args.reps, run)

    # the importance launch alone, with the arguments evaluate() built
    state, action, targets = imp._inputs(batch)
    variants, _, _ = imp.variants(A, S)
    ws = imp._bufs

    def eval_launch():
        imp._launch(state, action, targets, variants, ws)

    kern = [launch_us(eval_launch, args.launches) for _ in range(3)]
    fi, fs = results["fused"]
    ei, es = results["eager"]
    med = {k: v["median"] for k, v in per_eval.items()}
    return {"config": cfg, "variants": len(variants), "per_evaluate_us": per_eval,
            "speedup_median": med["eager"] / med["fused"],
            "eval_kernel_us": dict(median=statistics.median(kern), all=kern),
            "max_abs_diff_importance": float((torch.from_numpy(fi) - ei).abs().max()),
            "max_abs_diff_sensitivity": float((torch.from_numpy(fs) - es).abs().max()),
            "importance": fi.tolist(), "sensitivity": fs.tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the result file")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    args = ap.parse_args()

    dev = cuda_device(__file__)
    info = card_info()
    res = {
        "what": "FeatureImportanceEvaluator.evaluate + FeatureSensitivityEvaluator.evaluate vs "
                "the reference's per-feature loop in eager torch (cuDNN LSTM), per evaluation "
                "of both",
        "card": info,
        "method": (f"per shape, {args.reps} alternating repetitions of {args.iters} host-timed "
                   f"evaluations (synchronised before, each ending in its read-back) per "
                   f"variant after {args.warmup} warm-up evaluations; rb200_mdnrnn_eval of the "
                   f"1 + A + S importance variants: CUDA events over {args.launches} "
                   "back-to-back launches after 10 warm-up launches, 3 repetitions"),
        "shapes": {name: time_shape(name, cfg, args, dev) for name, cfg in SHAPES.items()},
    }
    write_result(args.out, __file__, res)


if __name__ == "__main__":
    main()
