"""TEST INFRASTRUCTURE ONLY -- float64 restatements of the row-local loss heads and the dueling
fold, taking the heads' inputs (network outputs, batch columns) instead of networks.

Each function restates the reference lines it cites; d loss / d head output comes from
torch.autograd in float64.  tests/test_loss_heads_cpu.py pins every function against
oracle/td_oracle.py (itself pinned to the unmodified reference) on the golden cases, and
tests/test_loss_heads_gpu.py compares the CUDA heads with them at the edges of their shapes.

Inputs may be any float tensors; they are cast to float64.  Optional inputs are None.  Every
function returns a dict with the outputs of the matching C entry point:
  loss, loss_partials, dz (and dz_reward / dz_qcpe for CPE), td_target, next_action_idx,
  all_q_values, propensities_next (CPE)."""
from typing import Optional

import torch
import torch.nn.functional as F

f64 = torch.float64
ACTION_NOT_POSSIBLE_VAL = -1e9


def _d(x):
    return None if x is None else torch.as_tensor(x).detach().to("cpu", f64)


def _discount(gamma, discount_src, B):
    """dqn_trainer.py:166-177 / c51_trainer.py:111-114: gamma ** discount_src or gamma."""
    if discount_src is None:
        return torch.full((B,), float(gamma), dtype=f64)
    return torch.pow(torch.tensor(float(gamma), dtype=f64), _d(discount_src).reshape(B))


def _boost(reward, action, reward_boost):
    """dqn_trainer_base.py:216-241"""
    if reward_boost is None:
        return reward
    return reward + (action * _d(reward_boost).reshape(1, -1)).sum(1)


def argmax_near_ties(values, rel=1e-5):
    """Rows whose two largest values lie within `rel` (relative to the larger magnitude): on
    those rows a float32 kernel may legitimately pick either action."""
    if values.shape[1] < 2:
        return torch.zeros(values.shape[0], dtype=torch.bool)
    top = values.topk(2, dim=1).values
    return (top[:, 0] - top[:, 1]) <= rel * top[:, 0].abs().clamp_min(1e-30)


def _pick(values, next_idx):
    """First arg max (torch.argmax); `next_idx` overrides it where not None (rows where the
    kernel's choice is fed back, see argmax_near_ties)."""
    idx = values.argmax(1)
    if next_idx is not None:
        idx = torch.as_tensor(next_idx).to("cpu", torch.int64).reshape(-1)
    return idx


# ---------------------------------------------------------------------------
# QR-DQN: reagent/training/qrdqn_trainer.py:108-155, :210-218
# ---------------------------------------------------------------------------
def qr_head(q_next_online, q_next_target, q_cur, action, next_action, mask, reward, not_terminal,
            *, num_atoms, gamma, double_q, maxq, discount_src=None, reward_boost=None,
            sample_weight=None, next_idx=None, row_chunk=512):
    """The quantile-Huber loss over the (N, B, N) pairs, computed over row chunks: the loss is
    a sum of row-local terms, so each chunk's autograd gives its rows' gradient."""
    q_cur, q_next_target = _d(q_cur), _d(q_next_target)
    B, N = q_cur.shape[0], num_atoms
    A = q_cur.shape[1] // N
    action = _d(action).reshape(B, A)
    reward = _boost(_d(reward).reshape(B), action, reward_boost)
    discount = _discount(gamma, discount_src, B)
    not_done = _d(not_terminal).reshape(B)
    quantiles = ((0.5 + torch.arange(N, dtype=f64)) / float(N)).view(1, -1)  # :70-73
    next_qf = q_next_target.view(B, A, N)  # :125
    out = {"next_action_idx": None}
    if maxq:  # :127-137
        sel = _d(q_next_online).view(B, A, N) if double_q else next_qf
        m = torch.ones(B, A, dtype=f64) if mask is None else _d(mask).reshape(B, A)
        qv = sel.mean(dim=2) + ACTION_NOT_POSSIBLE_VAL * (1 - m)  # :210-214
        idx = _pick(qv, next_idx)
        out["next_action_idx"], out["next_q_values"] = idx, qv
        next_qf = next_qf[torch.arange(B), idx]
    else:  # :139
        next_qf = (next_qf * _d(next_action).reshape(B, A).unsqueeze(-1)).sum(1)
    target = reward.view(B, 1) + discount.view(B, 1) * not_done.view(B, 1) * next_qf  # :142
    cur = q_cur.view(B, A, N).clone().requires_grad_(True)
    out["all_q_values"] = cur.detach().mean(2)  # :146
    w = None if sample_weight is None else _d(sample_weight).reshape(B)
    partials = torch.empty(B, dtype=f64)
    dz = torch.empty(B, A, N, dtype=f64)
    loss = torch.zeros((), dtype=f64)
    for r0 in range(0, B, row_chunk):
        rows = slice(r0, min(B, r0 + row_chunk))
        c = cur[rows]
        current = (c * action[rows].unsqueeze(-1)).sum(1)  # :149
        td = target[rows].t().unsqueeze(-1) - current  # (N, b, N), :152
        huber = torch.where(td.abs() < 1, 0.5 * td.pow(2), td.abs() - 0.5)  # :217-218
        per = (huber * (quantiles - (td.detach() < 0).to(f64)).abs()).sum(dim=(0, 2))  # :153-155
        scaled = per if w is None else per * w[rows]
        part = scaled.sum() / (N * B * N)
        (g,) = torch.autograd.grad(part, c)
        partials[rows], dz[rows] = per.detach(), g
        loss = loss + part.detach()
    out.update(loss=loss, loss_partials=partials, dz=dz.reshape(B, A * N), target=target)
    return out


# ---------------------------------------------------------------------------
# C51: reagent/training/c51_trainer.py:98-173, reagent/models/categorical_dqn.py:28-35
# ---------------------------------------------------------------------------
def c51_head(logits_next_online, logits_next_target, logits_cur, action, next_action, mask, reward,
             not_terminal, support, *, gamma, qmin, qmax, scale_support, double_q, maxq,
             discount_src=None, reward_boost=None, sample_weight=None, next_idx=None):
    """`support` and `scale_support` are the values the trainer hands the kernel (the reference
    builds them in float32 and Python floats).  Two places where the reference has no defined
    result take the kernel's reading, so that the rest of the batch can still be compared:
    a NaN target (the reference's scatter index is undefined) projects onto atom 0, and b is
    clamped to N - 1 (the reference indexes past m when (qmax - qmin) / scale_support > N - 1)."""
    lc = _d(logits_cur)
    B, N = lc.shape[0], support.shape[-1]
    A = lc.shape[1] // N
    support = _d(support).reshape(N)
    action = _d(action).reshape(B, A)
    reward = _boost(_d(reward).reshape(B), action, reward_boost)
    discount = _discount(gamma, discount_src, B)
    not_terminal = _d(not_terminal).reshape(B)
    next_dist = F.log_softmax(_d(logits_next_target).view(B, A, N), -1).exp()
    out = {"next_action_idx": None}
    if maxq:  # :117-129
        src = _d(logits_next_online) if double_q else _d(logits_next_target)
        next_q = (F.log_softmax(src.view(B, A, N), -1).exp() * support).sum(2)
        m_ = torch.ones(B, A, dtype=f64) if mask is None else _d(mask).reshape(B, A)
        qv = next_q + ACTION_NOT_POSSIBLE_VAL * (1 - m_)
        idx = _pick(qv, next_idx)
        out["next_action_idx"], out["next_q_values"] = idx, qv
        next_dist = next_dist[torch.arange(B), idx]
    else:  # :131-133
        next_dist = (next_dist * _d(next_action).reshape(B, A).unsqueeze(-1)).sum(1)
    target = (reward.view(B, 1) + discount.view(B, 1) * not_terminal.view(B, 1) * support)
    target = target.clamp(qmin, qmax)  # :135-139 (clamp keeps NaN)
    b = ((target - qmin) / float(scale_support)).clamp(max=N - 1)
    nan = b != b
    lo, up = b.floor(), b.ceil()
    lo[nan], up[nan] = 0, 0
    lo, up = lo.to(torch.int64), up.to(torch.int64)
    lo[(up > 0) * (lo == up)] -= 1  # :147-150
    up[(lo < (N - 1)) * (lo == up)] += 1
    m = torch.zeros_like(next_dist)
    m.scatter_add_(dim=1, index=lo, src=next_dist * (up.to(f64) - b))  # :152-160
    m.scatter_add_(dim=1, index=up, src=next_dist * (b - lo.to(f64)))
    cur = lc.view(B, A, N).clone().requires_grad_(True)
    log_dist = F.log_softmax(cur, -1)
    per = -(m * (log_dist * action.unsqueeze(-1)).sum(1)).sum(1)  # :162-168
    w = None if sample_weight is None else _d(sample_weight).reshape(B)
    loss = (per if w is None else per * w).mean()
    (dz,) = torch.autograd.grad(loss, cur)
    out.update(loss=loss.detach(), loss_partials=per.detach(), dz=dz.reshape(B, A * N), m=m,
               next_dist=next_dist,
               all_q_values=(log_dist.detach().exp() * support).sum(2))  # :170-171
    return out


# ---------------------------------------------------------------------------
# ParametricDQN: reagent/training/parametric_dqn_trainer.py:109-173,
# dqn_trainer_base.py:33-77 (get_max_q_values_with_target)
# ---------------------------------------------------------------------------
def _td_loss(q, target, loss):
    """dqn_trainer_base.py:146-155: mse | huber (smooth_l1) and d loss / d q."""
    q = q.clone().requires_grad_(True)
    fn = F.mse_loss if loss == "mse" else F.smooth_l1_loss
    value = fn(q, target)
    (dz,) = torch.autograd.grad(value, q)
    return value.detach(), dz


def pdqn_head(next_q, next_q_target, mask, reward, not_terminal, q_values, *, max_num_action,
              gamma, double_q, loss, discount_src=None):
    """max_num_action M > 0: masked (double-)max over the M tiled next actions of each row;
    M = 0: SARSA, next_q_target is q_target(s', next_action).  Double-Q needs next_q (without
    it the target net's own max is taken, as the kernel does)."""
    qv = _d(q_values)
    B, M = qv.numel(), max_num_action
    if M > 0:
        m = torch.ones(B, M, dtype=f64) if mask is None else _d(mask).reshape(B, M)
        pen = ACTION_NOT_POSSIBLE_VAL * (1 - m)  # dqn_trainer_base.py:59-62
        qtv = _d(next_q_target).reshape(B, M) + pen
        if double_q and next_q is not None:  # :64-75
            idx = (_d(next_q).reshape(B, M) + pen).argmax(1, keepdim=True)
            nq = torch.gather(qtv, 1, idx).reshape(B)
        else:
            nq = qtv.max(1).values
    else:
        nq = _d(next_q_target).reshape(B)
    # parametric_dqn_trainer.py:159: reward + not_terminal * discount * next_q
    target = _d(reward).reshape(B) + _d(not_terminal).reshape(B) * _discount(gamma, discount_src, B) * nq
    value, dz = _td_loss(qv.reshape(B), target, loss)
    return {"loss": value, "dz": dz, "td_target": target}


# ---------------------------------------------------------------------------
# CPE: dqn_trainer_base.py:332-452, reagent/core/torch_utils.py:62-73
# ---------------------------------------------------------------------------
def masked_softmax(x, mask, temperature):
    """torch_utils.py:62-73"""
    x = x / temperature
    mmx = x - ((1.0 - mask) * 1e20)
    mmx = mmx - torch.max(mmx, dim=1, keepdim=True)[0]
    e = torch.exp(mmx) * mask
    out = e / e.sum(dim=1, keepdim=True)
    out[out != out] = 0
    return out


def cpe_heads(next_scores, mask, action, metrics_reward, not_terminal, reward_est, qcpe,
              qcpe_target_next, *, temperature, gamma, loss, discount_src=None):
    """loss = (reward loss, CPE q-value loss); dz_reward / dz_qcpe: d loss / d network output
    [B, M*A]."""
    ns = _d(next_scores)
    B, A = ns.shape
    mrc = _d(metrics_reward).reshape(B, -1)
    M = mrc.shape[1]
    m = torch.ones(B, A, dtype=f64) if mask is None else _d(mask).reshape(B, A)
    offsets = torch.arange(0, M * A, A, dtype=torch.long)
    logged = torch.argmax(_d(action).reshape(B, A), dim=1, keepdim=True)  # :385
    prop = masked_softmax(ns, m, temperature)  # :387-391
    discount = _discount(gamma, discount_src, B).view(B, 1)
    not_done = _d(not_terminal).reshape(B, 1)
    r_all = _d(reward_est).reshape(B, M * A).clone().requires_grad_(True)
    r_loss = F.mse_loss(r_all.gather(1, offsets + logged), mrc)  # :392-399
    (dz_r,) = torch.autograd.grad(r_loss, r_all)
    c_all = _d(qcpe).reshape(B, M * A).clone().requires_grad_(True)
    metric_q = c_all.gather(1, offsets + logged)  # :404-406
    chunks = torch.chunk(_d(qcpe_target_next).reshape(B, M * A), M, dim=1)
    tgt = torch.cat([mrc[:, i:i + 1] + discount * ((ch * prop).sum(1, keepdim=True) * not_done)
                     for i, ch in enumerate(chunks)], dim=1)  # :407-423
    fn = F.mse_loss if loss == "mse" else F.smooth_l1_loss
    c_loss = fn(metric_q, tgt)  # :425-428
    (dz_c,) = torch.autograd.grad(c_loss, c_all)
    return {"loss": torch.stack([r_loss.detach(), c_loss.detach()]), "dz_reward": dz_r,
            "dz_qcpe": dz_c, "propensities_next": prop, "logged": logged.reshape(B)}


# ---------------------------------------------------------------------------
# Dueling head: reagent/models/dueling_q_network.py:92-103
# ---------------------------------------------------------------------------
def dueling_q(W_adv, b_adv, w_val, b_val, h_adv, h_val, num_actions, num_atoms):
    """q (rows, A*N) = value + (advantage - mean over actions and atoms of advantage) for head
    activations h_adv, h_val (rows, H)."""
    value = F.linear(h_val, w_val, b_val)  # (rows, N)
    adv = F.linear(h_adv, W_adv, b_adv).view(-1, num_actions, num_atoms)
    q = value.view(-1, 1, num_atoms) + (adv - adv.mean(dim=(1, 2), keepdim=True))
    return q.reshape(-1, num_actions * num_atoms)


def dueling_fold(W_adv, b_adv, w_val, b_val, num_actions, num_atoms):
    """The Linear [2H -> A*N] equal to the dueling head on h = [h_adv | h_val]: evaluated on
    h = 0 (bias) and on the 2H unit vectors (columns).  Differentiable in the true parameters,
    so its vector-Jacobian product is the transposed map the unfold applies."""
    H = W_adv.shape[1]
    eye = torch.eye(2 * H, dtype=W_adv.dtype)
    z = torch.zeros(1, 2 * H, dtype=W_adv.dtype)
    h = torch.cat([z, eye])
    q = dueling_q(W_adv, b_adv, w_val, b_val, h[:, :H], h[:, H:], num_actions, num_atoms)
    b_q = q[0]
    return (q[1:] - b_q).t(), b_q  # W_q [A*N, 2H], b_q [A*N]


def dueling_unfold(W_adv, b_adv, w_val, b_val, dW_q, db_q, num_actions, num_atoms):
    """d loss / d (W_adv, b_adv, w_val, b_val) given d loss / d (W_q, b_q)."""
    ps = [_d(p).requires_grad_(True) for p in (W_adv, b_adv, w_val, b_val)]
    W_q, b_q = dueling_fold(*ps, num_actions, num_atoms)
    return torch.autograd.grad((W_q, b_q), ps, (_d(dW_q), _d(db_q)))
