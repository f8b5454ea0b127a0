"""The world-model evaluator goldens (tests/golden/wm_eval_*.npz) as the oracle reads them,
shared by the CPU and GPU tests."""
import numpy as np
import torch

from oracle import mdnrnn_oracle as mo
from oracle import world_model_eval_oracle as wo

CASES = ["wm_eval_cartpole_features", "wm_eval_defaults_t16", "wm_eval_continuous_groups",
         "wm_eval_fit_last_terminal"]
TOL = 1e-5


def cfg_of(meta):
    return dict(L=meta["L"], G=meta["G"], next_state_weight=meta["next_state_weight"],
                not_terminal_weight=meta["not_terminal_weight"],
                reward_weight=meta["reward_weight"],
                fit_only_one_next_step=meta["fit_only_one_next_step"])


def params64(arrays, meta):
    p = mo.initial_params(meta["seed"], meta["S"], meta["A"], meta["H"], meta["L"], meta["G"])
    for i, t in enumerate(p):
        np.testing.assert_array_equal(mo.digest(t), arrays[f"p0.{i}.sha256"], err_msg=f"p0.{i}")
    return [t.double() for t in p]


def batch_of(arrays, dtype=torch.float64):
    return {k: torch.from_numpy(arrays[f"batch.{k}"]).to(dtype)
            for k in ("state", "action", "next_state", "reward", "not_terminal")}


def sensitivity_tol(arrays, meta):
    """The tolerance of each state feature's sensitivity: TOL times the mean over (T, B, G) of
    the feature's sum of |mu| of both forwards.  A sensitivity is a mean of differences of
    means, so its rounding error scales with the means, not with their difference."""
    P = params64(arrays, meta)
    b = batch_of(arrays)
    perm = torch.from_numpy(arrays["perm"])
    m0 = mo.forward(P, b["state"], b["action"], meta["L"], meta["G"])["mus"]
    m1 = mo.forward(P, b["state"], b["action"][:, perm], meta["L"], meta["G"])["mus"]
    return np.array([float((m0[..., s:e].abs() + m1[..., s:e].abs()).sum(dim=3).mean()) * TOL
                     for s, e in wo.groups(meta["state_starts"], meta["S"])])


def importance_of(arrays, meta):
    return wo.feature_importance(params64(arrays, meta), batch_of(arrays), cfg_of(meta),
                                 discrete_action=meta["discrete"],
                                 action_starts=meta["action_starts"],
                                 state_starts=meta["state_starts"])
