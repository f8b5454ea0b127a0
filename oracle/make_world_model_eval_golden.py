"""Generate the world-model evaluator golden vectors tests/golden/wm_eval_*.npz by running the
UNMODIFIED reference FeatureImportanceEvaluator and FeatureSensitivityEvaluator
(reagent/evaluation/world_model_evaluator.py) through oracle/ref_harness.py, on a seeded
MemoryNetwork (its weights are oracle.mdnrnn_oracle.initial_params(seed, ...)) and a seeded
batch.  Needs the reference checkout; the files are committed.

    python oracle/make_world_model_eval_golden.py            # every case
    python oracle/make_world_model_eval_golden.py NAME ...   # only the named ones

A case holds
  p0.{i}.sha256     SHA-256 of the initial parameters, parameters() order
  batch.{state,action,next_state,reward,not_terminal}
  losses            [1 + A_feat + S_feat, 4] (gmm, bce, mse, loss) of every get_loss call of
                    the importance evaluator, in call order (the original batch first)
  fill.{v}          the value variant v >= 1 wrote into its columns (the one-hot e_i of a
                    discrete action, else compute_median_feature_value's result)
  increase          feature_loss_increase
  perm              the torch.randperm(B) the sensitivity evaluator drew after
                    torch.manual_seed(meta["perm_seed"])
  sensitivity       feature_sensitivity
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden import _np, _save  # noqa: E402
from oracle.make_mdnrnn_golden import _batch  # noqa: E402
from oracle.mdnrnn_oracle import digest, initial_params  # noqa: E402
from oracle.ref_harness import ref  # noqa: E402

LOSS_KEYS = ("gmm", "bce", "mse", "loss")


def _enum(gen, counts):
    """One-hot rows [sum(counts), len(counts)] with exactly counts[k] rows of category k, in a
    seeded order."""
    cat = torch.cat([torch.full((c,), k, dtype=torch.int64) for k, c in enumerate(counts)])
    cat = cat[torch.randperm(cat.numel(), generator=gen)]
    return torch.nn.functional.one_hot(cat, len(counts)).float()


def _grouped_batch(gen, T, B, S, A, p_terminal, state_enums, action_enums):
    """_batch, then the columns of each (first column, counts) enum replaced by one-hots."""
    b = _batch(gen, T, B, S, A, False, p_terminal)
    for key, enums, dim in (("state", state_enums, S), ("action", action_enums, A)):
        x = b[key].reshape(T * B, dim)
        for c0, counts in enums:
            x[:, c0:c0 + len(counts)] = _enum(gen, counts)
        b[key] = x.reshape(T, B, dim)
    return b


def case(name, *, S, A, T, B, discrete, action_starts, state_starts, p_terminal=0.05,
         seed=0, state_enums=(), action_enums=(), **param_kw):
    rlt = ref("reagent.core.types")
    params_mod = ref("reagent.core.parameters")
    wm = ref("reagent.models.world_model")
    trainer_mod = ref("reagent.training.world_model.mdnrnn_trainer")
    ev = ref("reagent.evaluation.world_model_evaluator")
    params = params_mod.MDNRNNTrainerParameters(action_dim=A, **param_kw)
    torch.manual_seed(seed)
    net = wm.MemoryNetwork(state_dim=S, action_dim=A, num_hiddens=params.hidden_size,
                           num_hidden_layers=params.num_hidden_layers,
                           num_gaussians=params.num_gaussians)
    trainer = trainer_mod.MDNRNNTrainer(memory_network=net, params=params)
    trainer.trainer = None
    arrays = {}
    p0 = initial_params(seed, S, A, params.hidden_size, params.num_hidden_layers,
                        params.num_gaussians)
    for i, p in enumerate(net.mdnrnn.parameters()):
        assert torch.equal(p.detach(), p0[i]), (name, i)
        arrays[f"p0.{i}.sha256"] = digest(p)

    gen = torch.Generator().manual_seed(seed + 1000)
    if state_enums or action_enums:
        b = _grouped_batch(gen, T, B, S, A, p_terminal, state_enums, action_enums)
    else:
        b = _batch(gen, T, B, S, A, discrete, p_terminal)
    for k, v in b.items():
        arrays[f"batch.{k}"] = _np(v).copy()
    batch = rlt.MemoryNetworkInput(
        state=rlt.FeatureData(float_features=b["state"]),
        next_state=rlt.FeatureData(float_features=b["next_state"]),
        action=rlt.FeatureData(float_features=b["action"]), reward=b["reward"],
        not_terminal=b["not_terminal"], time_diff=None, step=None)

    # feature importance, recording every get_loss and every fill value
    a_feat = A if discrete else len(action_starts)
    imp = ev.FeatureImportanceEvaluator(
        trainer, discrete_action=discrete, state_feature_num=len(state_starts),
        action_feature_num=a_feat, sorted_action_feature_start_indices=list(action_starts),
        sorted_state_feature_start_indices=list(state_starts))
    losses, fills = [], []
    get_loss = trainer.get_loss

    def recording_get_loss(*args, **kw):
        out = get_loss(*args, **kw)
        losses.append([float(out[k]) for k in LOSS_KEYS])
        return out

    median = imp.compute_median_feature_value

    def recording_median(features):
        out = median(features)
        fills.append(out.detach().clone())
        return out

    trainer.get_loss = recording_get_loss
    imp.compute_median_feature_value = recording_median
    with torch.no_grad():
        increase = imp.evaluate(batch)["feature_loss_increase"]
    del trainer.get_loss
    if discrete:
        fills = [torch.eye(A)[i] for i in range(A)] + fills
    assert len(losses) == 1 + a_feat + len(state_starts) == 1 + len(fills)
    arrays["losses"] = np.array(losses, dtype=np.float64)
    for v, f in enumerate(fills, start=1):
        arrays[f"fill.{v}"] = _np(f).copy()
    arrays["increase"] = np.asarray(increase).copy()

    # feature sensitivity, recording the permutation
    sens = ev.FeatureSensitivityEvaluator(trainer, state_feature_num=len(state_starts),
                                          sorted_state_feature_start_indices=list(state_starts))
    randperm, drawn = torch.randperm, []

    def recording_randperm(*args, **kw):
        p = randperm(*args, **kw)
        drawn.append(p.clone())
        return p

    perm_seed = seed + 7
    torch.manual_seed(perm_seed)
    torch.randperm = recording_randperm
    try:
        with torch.no_grad():
            sensitivity = sens.evaluate(batch)["feature_sensitivity"]
    finally:
        torch.randperm = randperm
    assert len(drawn) == 1
    arrays["perm"] = _np(drawn[0]).copy()
    arrays["sensitivity"] = np.asarray(sensitivity).copy()

    meta = dict(kind="wm_eval", S=S, A=A, T=T, B=B, H=params.hidden_size,
                L=params.num_hidden_layers, G=params.num_gaussians,
                next_state_weight=params.next_state_loss_weight,
                not_terminal_weight=params.not_terminal_loss_weight,
                reward_weight=params.reward_loss_weight,
                fit_only_one_next_step=params.fit_only_one_next_step, discrete=discrete,
                action_starts=list(action_starts), state_starts=list(state_starts),
                action_feature_num=a_feat, seed=seed, perm_seed=perm_seed)
    _save(name, arrays, meta)


CASES = [
    # configs/world_model/cartpole_features.yaml at a batch that is not a multiple of 16
    ("wm_eval_cartpole_features", dict(S=4, A=2, T=1, B=1000, discrete=True,
                                       action_starts=[0, 1], state_starts=[0, 1, 2, 3],
                                       hidden_size=50, num_hidden_layers=2, num_gaussians=1,
                                       seed=0)),
    # MDNRNNTrainerParameters() defaults (hidden 64, 2 layers, 5 gaussians) over 16 steps
    ("wm_eval_defaults_t16", dict(S=4, A=2, T=16, B=150, discrete=True, action_starts=[0, 1],
                                  state_starts=[0, 1, 2, 3], p_terminal=0.1, seed=2)),
    # continuous action; width-1 columns mixed with enum one-hot groups: a 4-column group with
    # a tie at the lower median, a 3-column group, and a 2-column action group whose lower and
    # upper medians differ
    ("wm_eval_continuous_groups", dict(S=10, A=3, T=3, B=33, discrete=False,
                                       action_starts=[0, 1], state_starts=[0, 1, 5, 6, 9],
                                       state_enums=((1, (20, 49, 10, 20)), (6, (15, 40, 44))),
                                       action_enums=((1, (59, 40)),), hidden_size=32,
                                       num_hidden_layers=1, num_gaussians=2, seed=4)),
    # loss on the last step only, with terminal rows
    ("wm_eval_fit_last_terminal", dict(S=3, A=1, T=4, B=97, discrete=False, action_starts=[0],
                                       state_starts=[0, 1, 2], p_terminal=0.3, hidden_size=37,
                                       num_hidden_layers=3, num_gaussians=3,
                                       fit_only_one_next_step=True, seed=3)),
]


def main(only=None):
    for name, kw in CASES:
        if not only or name in only:
            case(name, **kw)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
