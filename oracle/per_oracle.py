"""Prioritized experience replay (Schaul et al. 2016) on top of td_oracle: the weighted DQN
update, the TD-error priorities, the importance weights and the beta schedule that
FusedDqnStep(per=PrioritizedUpdate(...)) computes on the GPU.  The reference documents this
(SumTree / PrioritizedReplayBuffer.set_priority docstrings) but never wires it up, so there is no
reference golden for it; with w = 1 the update is td_oracle.dqn_update, which is pinned to the
reference's goldens."""
import numpy as np
import torch
import torch.nn.functional as F

from . import bcq_oracle as BO
from . import td_oracle as O


def weighted_td_loss(q, qt, batch, weights, *, gamma, loss="mse", imitator=None,
                     bcq_threshold=None, maxq=True, **kw):
    """mean_i(w_i * loss_i) with the per-row DQN loss of dqn_trainer.py:229-238; with an
    imitator, the max-Q next-action mask is narrowed by the BCQ filter (bcq_oracle)."""
    if imitator is not None and maxq:
        batch = dict(batch, possible_next_actions_mask=BO.filtered_next_mask(batch, imitator,
                                                                             bcq_threshold))
    _, aux = O.dqn_td_loss(q, qt, batch, gamma=gamma, loss=loss, maxq=maxq, **kw)
    q_sel = torch.sum(O.mlp(q, batch["state"]) * batch["action"], 1, keepdim=True)
    fn = F.mse_loss if loss == "mse" else F.smooth_l1_loss
    rows = fn(q_sel, aux["target"], reduction="none").reshape(-1)
    return torch.mean(weights.reshape(-1) * rows), aux


def weighted_dqn_update(q, qt, adam, batch, weights, *, gamma, tau, **kw):
    """dqn_update with the importance-weighted TD loss.  Returns (loss, grads, aux)."""
    params = O.net_params(q)
    for p in params:
        p.grad = None
    loss, aux = weighted_td_loss(q, qt, batch, weights, gamma=gamma, **kw)
    loss.backward()
    grads = [p.grad.detach().clone() for p in params]
    adam.step(params, grads)
    O.soft_update(qt, q, tau)
    return float(loss.detach()), grads, aux


def priorities(q_selected, td_target, alpha, eps):
    """p_i = ((double)|q_selected_i - td_target_i| + eps) ** alpha; the difference in fp32."""
    d = np.abs(np.asarray(q_selected, np.float32) - np.asarray(td_target, np.float32))
    return (d.astype(np.float64) + eps) ** alpha


def beta(t, beta0, beta_updates):
    """beta_t = min(1, beta0 + (1 - beta0) * t / beta_updates)."""
    return min(1.0, beta0 + (1.0 - beta0) * t / beta_updates)


def importance_weights(leaves, beta_t):
    """w_i = (p_min / p_i) ** beta_t over the drawn leaves (fp64); a zero leaf gets w = 0 and is
    left out of p_min.  The buffer size and the tree total cancel in this normalisation."""
    leaves = np.asarray(leaves, np.float64)
    pos = leaves > 0.0
    if not pos.any():
        return np.zeros_like(leaves)
    p_min = leaves[pos].min()
    w = np.zeros_like(leaves)
    w[pos] = (p_min / leaves[pos]) ** beta_t
    return w
