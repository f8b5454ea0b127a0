"""Prioritized replay for the distributional heads, on top of td_oracle and per_oracle: the
importance-weighted QR-DQN and C51 updates and the row-loss priorities that
FusedDqnStep(per=PrioritizedUpdate(...)) computes on the GPU for QRDQNTrainer and C51Trainer.

These heads have no scalar TD error, so a row's priority is its own distributional loss (as in
Rainbow and Dopamine's quantile / Rainbow agents).  The per-row losses restate
td_oracle.qrdqn_loss / c51_loss without their batch mean; with w = 1 the weighted updates reduce
to td_oracle.qrdqn_update / c51_update, which are pinned to the reference's goldens.  The
reference never wires prioritized replay, so there is no golden of the weighted update itself."""
import numpy as np
import torch
import torch.nn.functional as F

from . import td_oracle as O


def _reward_discount(batch, gamma, discount_src, reward_boost):
    reward, action = batch["reward"], batch["action"]
    if reward_boost is not None:
        reward = reward + torch.sum(action.float() * reward_boost, dim=1, keepdim=True)
    discount = torch.full_like(reward, gamma)
    if discount_src is not None:
        discount = torch.pow(gamma, discount_src.float())
    return reward, discount


def qrdqn_row_loss(q, qt, batch, *, gamma, num_atoms, double_q=True, maxq=True,
                   discount_src=None, reward_boost=None):
    """[B] per-row QR-DQN losses: td_oracle.qrdqn_loss's (N, B, N) quantile-Huber terms averaged
    over row b's N^2 atom pairs (i, j), without the mean over rows.  Returns (rows, aux)."""
    action = batch["action"]
    B, A, N = action.shape[0], action.shape[1], num_atoms
    reward, discount = _reward_discount(batch, gamma, discount_src, reward_boost)
    not_done = batch["not_terminal"].float()
    quantiles = ((0.5 + torch.arange(N).float()) / float(N)).view(1, -1)
    next_qf = O.mlp(qt, batch["next_state"]).view(B, A, N)
    if maxq:
        sel = O.mlp(q, batch["next_state"]).view(B, A, N) if double_q else next_qf
        qv = sel.mean(dim=2) + O.ACTION_NOT_POSSIBLE_VAL * (
            1 - batch["possible_next_actions_mask"].float())
        next_action = qv.argmax(1)
        next_qf = next_qf[range(B), next_action.reshape(-1)]
    else:
        next_action = None
        next_qf = (next_qf * batch["next_action"].unsqueeze(-1)).sum(1)
    target_Q = (reward + discount * not_done * next_qf).detach()
    current_qf = O.mlp(q, batch["state"]).view(B, A, N)
    all_q = current_qf.mean(2).detach()
    current_qf = (current_qf * action.unsqueeze(-1)).sum(1)
    td = target_Q.t().unsqueeze(-1) - current_qf  # (N, B, N)
    huber = torch.where(td.abs() < 1, 0.5 * td.pow(2), td.abs() - 0.5)
    rows = (huber * (quantiles - (td.detach() < 0).float()).abs()).mean(dim=(0, 2))
    return rows, {"next_action": next_action, "all_q": all_q, "target": target_Q}


def c51_row_loss(q, qt, batch, *, gamma, num_atoms, qmin, qmax, double_q=True, maxq=True,
                 discount_src=None, reward_boost=None):
    """[B] per-row C51 losses: -sum_c m_c log p_c(a_b), td_oracle.c51_loss without the mean over
    rows."""
    action = batch["action"]
    B, A, N = action.shape[0], action.shape[1], num_atoms
    support = torch.linspace(qmin, qmax, N)
    scale_support = (qmax - qmin) / (N - 1.0)
    reward, discount = _reward_discount(batch, gamma, discount_src, reward_boost)
    not_terminal = batch["not_terminal"].float()
    log_dist = lambda net, x: F.log_softmax(O.mlp(net, x).view(B, A, N), -1)  # noqa: E731
    with torch.no_grad():
        next_dist = log_dist(qt, batch["next_state"]).exp()
        if maxq:
            if double_q:
                next_q = (log_dist(q, batch["next_state"]).exp() * support).sum(2)
            else:
                next_q = (next_dist * support).sum(2)
            mask = batch["possible_next_actions_mask"].float()
            next_action = (next_q + O.ACTION_NOT_POSSIBLE_VAL * (1 - mask)).argmax(1)
            next_dist = next_dist[range(B), next_action.reshape(-1)]
        else:
            next_dist = (next_dist * batch["next_action"].unsqueeze(-1)).sum(1)
        target_Q = (reward + discount * not_terminal * support).clamp(qmin, qmax)
        b = (target_Q - qmin) / scale_support
        lo, up = b.floor().to(torch.int64), b.ceil().to(torch.int64)
        lo[(up > 0) * (lo == up)] -= 1
        up[(lo < (N - 1)) * (lo == up)] += 1
        m = torch.zeros_like(next_dist)
        m.scatter_add_(dim=1, index=lo, src=next_dist * (up.float() - b))
        m.scatter_add_(dim=1, index=up, src=next_dist * (b - lo.float()))
    ld = (log_dist(q, batch["state"]) * action.unsqueeze(-1)).sum(1)
    return -(m * ld).sum(1)


def _weighted_step(q, qt, adam, rows, weights, tau):
    params = O.net_params(q)
    loss = torch.mean(weights.reshape(-1) * rows)
    grads = [g.detach().clone() for g in torch.autograd.grad(loss, params)]
    adam.step(params, grads)
    O.soft_update(qt, q, tau)
    return float(loss.detach()), grads


def weighted_qrdqn_update(q, qt, adam, batch, weights, *, gamma, tau, num_atoms, **kw):
    """qrdqn_update with loss = mean_b(w_b * row_b).  Returns (loss, grads, aux); aux["rows"] holds
    the unweighted per-row losses, computed before the update."""
    rows, aux = qrdqn_row_loss(q, qt, batch, gamma=gamma, num_atoms=num_atoms, **kw)
    aux["rows"] = rows.detach().clone()
    loss, grads = _weighted_step(q, qt, adam, rows, weights, tau)
    return loss, grads, aux


def weighted_c51_update(q, qt, adam, batch, weights, *, gamma, tau, **kw):
    """c51_update with loss = mean_b(w_b * row_b).  Returns (loss, grads, rows), rows being the
    unweighted per-row cross entropies before the update."""
    rows = c51_row_loss(q, qt, batch, gamma=gamma, **kw)
    detached = rows.detach().clone()
    loss, grads = _weighted_step(q, qt, adam, rows, weights, tau)
    return loss, grads, detached


def row_loss_priorities(row_loss, divisor, alpha, eps):
    """p_b = ((double)|row_loss_b| / divisor + eps) ** alpha, in fp64 (divisor N^2 for the QR-DQN
    head's row sums, 1 for C51)."""
    r = np.abs(np.asarray(row_loss, np.float32).astype(np.float64))
    return (r / float(divisor) + eps) ** alpha
