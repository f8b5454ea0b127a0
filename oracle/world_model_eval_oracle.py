"""Plain-torch restatement of the world-model evaluators (reagent/evaluation/
world_model_evaluator.py FeatureImportanceEvaluator and FeatureSensitivityEvaluator) on
oracle/mdnrnn_oracle.py, in the dtype of its inputs (fp64 for the tests).

`batch`: state, action, next_state, reward, not_terminal ([T, B, ...]).  `cfg`: L, G and the
loss settings of mdnrnn_oracle.losses (next_state_weight, not_terminal_weight, reward_weight,
fit_only_one_next_step).
"""
import torch

from oracle import mdnrnn_oracle as mo


def groups(starts, dim):
    """[(begin, end)] of the features starting at `starts` in a vector of `dim` columns."""
    b = list(starts) + [dim]
    return list(zip(b[:-1], b[1:]))


def fill_value(features):
    """compute_median_feature_value of [N, w] features: the column mean for w == 1, else the
    one-hot at the first column whose column sum equals the lower median of the column sums."""
    if features.shape[1] > 1:
        counts = features.sum(dim=0)
        med = torch.sort(counts).values[(counts.numel() - 1) // 2]
        first = int(torch.nonzero(counts == med)[0, 0])
        out = torch.zeros(features.shape[1], dtype=features.dtype)
        out[first] = 1
        return out
    return features.mean(dim=0)


def _loss(params, batch, cfg, state=None, action=None):
    S = batch["state"].shape[2]
    out = mo.forward(params, batch["state"] if state is None else state,
                     batch["action"] if action is None else action, cfg["L"], cfg["G"])
    return mo.losses(out, batch["next_state"], batch["reward"], batch["not_terminal"],
                     next_state_weight=cfg["next_state_weight"],
                     not_terminal_weight=cfg["not_terminal_weight"],
                     reward_weight=cfg["reward_weight"],
                     fit_only_one_next_step=cfg["fit_only_one_next_step"], state_dim=S)


def feature_importance(params, batch, cfg, *, discrete_action, action_starts, state_starts):
    """{"losses": [1 + A_feat + S_feat, 4] (gmm, bce, mse, loss) of the original batch and
    of each variant, "fills": the fill value of each variant ([] for the original), and
    "increase": loss_v - loss_0}."""
    T, B, S = batch["state"].shape
    A = batch["action"].shape[2]
    losses = [_loss(params, batch, cfg)]
    fills = [None]
    if discrete_action:
        a_groups = [(0, A)] * A
    else:
        a_groups = groups(action_starts, A)
    for i, (b, e) in enumerate(a_groups):
        act = batch["action"].reshape(T * B, A).clone()
        if discrete_action:
            f = torch.zeros(A, dtype=act.dtype)
            f[i] = 1
        else:
            f = fill_value(act[:, b:e])
        act[:, b:e] = f
        fills.append(f)
        losses.append(_loss(params, batch, cfg, action=act.reshape(T, B, A)))
    for b, e in groups(state_starts, S):
        st = batch["state"].reshape(T * B, S).clone()
        f = fill_value(st[:, b:e])
        st[:, b:e] = f
        fills.append(f)
        losses.append(_loss(params, batch, cfg, state=st.reshape(T, B, S)))
    tab = torch.stack([torch.stack([ls[k] for k in mo.LOSS_KEYS]) for ls in losses])
    return {"losses": tab, "fills": fills, "increase": tab[1:, 3] - tab[0, 3]}


def feature_sensitivity(params, batch, cfg, *, state_starts, perm):
    """Per state feature: mean over (T, B, G) of sum over its columns of |mus(shuffled actions)
    - mus(actions)|, the actions shuffled along the batch by `perm`."""
    S = batch["state"].shape[2]
    mus0 = mo.forward(params, batch["state"], batch["action"], cfg["L"], cfg["G"])["mus"]
    mus1 = mo.forward(params, batch["state"], batch["action"][:, perm, :], cfg["L"],
                      cfg["G"])["mus"]
    return torch.stack([(mus1[..., b:e] - mus0[..., b:e]).abs().sum(dim=3).mean()
                        for b, e in groups(state_starts, S)])
