"""Discrete CRR (reagent/training/discrete_crr_trainer.py) restated in plain torch: the readable
specification of one DiscreteCRRTrainer update, the CPU side of the parity tests, and -- run in
float64 -- the reference of the two loss heads in reagent_b200/csrc/rb200_crr.cu.

Per batch, in the order of the reference's generator:
  1. y = boosted reward + gamma * V' * not_terminal, V' = sum_a softmax(l')_a q1_target(s')_a
     (min with q2_target's), l' the actor's (or target actor's) output on s'
  2. q1 <- Adam(mse(q1(s, a), y)); q2 likewise, on the same y
  3. with the UPDATED q1: weight = clamp(exp((q1(s, a) - V) / beta), 0, max_weight), a constant;
     actor <- Adam(mean(-log pi(a) * weight) [+ entropy_coeff * mean(ratio * log pi(a))]) on
     every `delayed_policy_update`-th batch
  4. the CPE networks (next-state propensities from q1_target(s') of step 1)
  5. the soft update of every target, on every batch
The actor's output is FullyConnectedActor.forward's (reagent/models/actor.py:90-110): act(z),
and with exploration noise clamp(act(z) + noise, -1, 1).
"""
import torch
import torch.nn.functional as F

from oracle import td_oracle as O


def actor_logits(actor_out, noise):
    return actor_out if noise is None else (actor_out + noise).clamp(-1.0, 1.0)


def td_target(l_next, q1t_next, q2t_next, reward, action, reward_boost, not_terminal, gamma):
    """compute_target_q_values (:198-212) after boost_rewards (dqn_trainer_base.py:216-241);
    reward / not_terminal are [B, 1], reward_boost [1, A] or None."""
    p = F.softmax(l_next, dim=1)
    v = (q1t_next * p).sum(dim=1, keepdim=True)
    if q2t_next is not None:
        v = torch.min(v, (q2t_next * p).sum(dim=1, keepdim=True))
    if reward_boost is not None:
        reward = reward + (action * reward_boost).sum(dim=1, keepdim=True)
    return reward + gamma * v * not_terminal


def td_loss(q, action, y):
    """compute_td_loss (:214-218)"""
    return F.mse_loss((q * action).sum(dim=1, keepdim=True), y)


def actor_losses(l, q, action, logged_prob, *, beta, max_weight, entropy_coeff, clip_limit):
    """compute_actor_loss (:220-288): (actor_loss_without_reg, actor_loss, weight [B, 1])."""
    a = torch.argmax(action, dim=1, keepdim=True)
    p = F.softmax(l, dim=1)
    log_pi = F.log_softmax(l, dim=1).gather(1, a)
    v = (q * p).sum(dim=1, keepdim=True)
    adv = ((q - v) * action).sum(dim=1, keepdim=True)
    weight = torch.clamp(((1 / beta) * adv).exp(), 0, max_weight).detach()
    without_reg = (-log_pi * weight).mean()
    loss = without_reg
    if entropy_coeff > 0:
        pi_t = (p * action).sum(dim=1, keepdim=True)
        ratio = torch.clip(pi_t / logged_prob.view(pi_t.shape), min=1e-4, max=clip_limit)
        loss = without_reg + entropy_coeff * (ratio * log_pi).mean()
    return without_reg, loss, weight


# ---------------------------------------------------------------------------
# float64 references of rb200_crr_critic_head / rb200_crr_actor_head
# ---------------------------------------------------------------------------
def _d(t):
    return None if t is None else torch.as_tensor(t).detach().double().cpu()


def critic_head_fp64(actor_next, noise_next, q1t_next, q2t_next, q1, q2, action, reward,
                     reward_boost, not_terminal, gamma):
    """reward / not_terminal [B], reward_boost [A] or None.  Returns y [B], q_sel (per critic),
    loss (per critic) and dz (per critic, d loss / d q)."""
    action = _d(action)
    y = td_target(actor_logits(_d(actor_next), _d(noise_next)), _d(q1t_next), _d(q2t_next),
                  _d(reward).view(-1, 1), action,
                  None if reward_boost is None else _d(reward_boost).view(1, -1),
                  _d(not_terminal).view(-1, 1), gamma)
    out = {"y": y.view(-1), "q_sel": [], "loss": [], "dz": []}
    for q in (q1, q2):
        if q is None:
            continue
        q = _d(q).requires_grad_(True)
        loss = td_loss(q, action, y)
        out["q_sel"].append((q.detach() * action).sum(dim=1))
        out["loss"].append(float(loss.detach()))
        out["dz"].append(torch.autograd.grad(loss, q)[0])
    return out


_ACT_BWD = {
    "linear": lambda y: torch.ones_like(y),
    "relu": lambda y: (y > 0).double(),
    "tanh": lambda y: 1 - y * y,
    "leaky_relu": lambda y: torch.where(y > 0, 1.0, 0.01).double(),
    "sigmoid": lambda y: y * (1 - y),
    "softplus": lambda y: 1 - torch.exp(-y),
}


def actor_head_fp64(actor_out, noise, q1, action, logged_prob, *, beta, max_weight,
                    entropy_coeff, clip_limit, activation="tanh"):
    """Returns loss (without_reg, with), weight [B] and dz = d loss / d z where
    actor_out = activation(z): autograd through the clamp, the softmax and the clipped ratio,
    times the activation's derivative written in terms of its output."""
    y = _d(actor_out).requires_grad_(True)
    wo, loss, w = actor_losses(actor_logits(y, _d(noise)), _d(q1), _d(action), _d(logged_prob),
                               beta=beta, max_weight=max_weight, entropy_coeff=entropy_coeff,
                               clip_limit=clip_limit)
    g = torch.autograd.grad(loss, y)[0]
    return {"loss": (float(wo.detach()), float(loss.detach())), "weight": w.view(-1),
            "dz": g * _ACT_BWD[activation](y.detach())}


# ---------------------------------------------------------------------------
# one update
# ---------------------------------------------------------------------------
class CrrState:
    """Networks as td_oracle nets ({"W", "b", "act"} or a dueling dict); the actor's last
    activation is its action_activation.  `make_adam(params)` builds each optimizer state."""

    def __init__(self, actor, actor_t, q1, q1_t, q2=None, q2_t=None, reward=None, qcpe=None,
                 qcpe_t=None, *, make_adam_q, make_adam_actor):
        self.actor, self.actor_t = actor, actor_t
        self.q1, self.q1_t, self.q2, self.q2_t = q1, q1_t, q2, q2_t
        self.reward, self.qcpe, self.qcpe_t = reward, qcpe, qcpe_t
        self.adam_q1 = make_adam_q(O.net_params(q1))
        self.adam_q2 = None if q2 is None else make_adam_q(O.net_params(q2))
        self.adam_actor = make_adam_actor(O.net_params(actor))
        self.adam_reward = None if reward is None else make_adam_q(O.net_params(reward))
        self.adam_qcpe = None if qcpe is None else make_adam_q(O.net_params(qcpe))


def crr_update(st: CrrState, batch, batch_idx: int, *, gamma, tau, noise_next=None,
               noise_cur=None, use_target_actor=False, delayed_policy_update=1, beta=1.0,
               entropy_coeff=0.0, clip_limit=10.0, max_weight=20.0, reward_boost=None,
               temperature=0.01, cpe_loss="mse"):
    """One update on `batch` (dict: state, next_state, action one-hot, reward [B,1],
    not_terminal [B,1], action_probability [B,1], possible_next_actions_mask, metrics).
    Returns (losses in yield order without the soft update's, None for a skipped actor step;
    grads per optimizer in the same order; the actor weights or None)."""
    s, s2, action = batch["state"], batch["next_state"], batch["action"]
    losses, grads = [], []
    with torch.no_grad():
        next_q = O.mlp(st.q1_t, s2)
        l_next = actor_logits(O.mlp(st.actor_t if use_target_actor else st.actor, s2), noise_next)
        y = td_target(l_next, next_q, None if st.q2 is None else O.mlp(st.q2_t, s2),
                      batch["reward"], action, reward_boost, batch["not_terminal"], gamma)
    for q, adam in ((st.q1, st.adam_q1), (st.q2, st.adam_q2)):
        if q is None:
            continue
        loss = td_loss(O.mlp(q, s), action, y)
        grads.append(O._grad_step(loss, q, adam))
        losses.append(float(loss.detach()))
    weight = None
    if batch_idx % delayed_policy_update == 0:
        with torch.no_grad():
            all_q = O.mlp(st.q1, s)
        _, loss, weight = actor_losses(
            actor_logits(O.mlp(st.actor, s), noise_cur), all_q, action,
            batch["action_probability"], beta=beta, max_weight=max_weight,
            entropy_coeff=entropy_coeff, clip_limit=clip_limit)
        grads.append(O._grad_step(loss, st.actor, st.adam_actor))
        losses.append(float(loss.detach()))
    else:
        grads.append(None)
        losses.append(None)
    if st.reward is not None:
        rl, cl = cpe_losses(st, batch, next_q, gamma=gamma, temperature=temperature,
                            loss=cpe_loss)
        grads.append(O._grad_step(rl, st.reward, st.adam_reward))
        grads.append(O._grad_step(cl, st.qcpe, st.adam_qcpe))
        losses += [float(rl.detach()), float(cl.detach())]
        O.soft_update(st.qcpe_t, st.qcpe, tau)
    O.soft_update(st.q1_t, st.q1, tau)
    if st.q2 is not None:
        O.soft_update(st.q2_t, st.q2, tau)
    O.soft_update(st.actor_t, st.actor, tau)
    return losses, grads, weight


def cpe_losses(st: CrrState, batch, next_q, *, gamma, temperature, loss="mse"):
    """_calculate_cpes (dqn_trainer_base.py:332-452) as DiscreteCRRTrainer calls it: the
    next-state propensities are masked_softmax(q1_target(s')), the discount is gamma."""
    A = batch["action"].shape[1]
    mrc = batch["reward"]
    if batch.get("metrics") is not None:
        mrc = torch.cat((batch["reward"], batch["metrics"]), dim=1)
    M = mrc.shape[1]
    idx = torch.arange(0, M * A, A) + torch.argmax(batch["action"], dim=1, keepdim=True)
    prop = O.masked_softmax(next_q, batch["possible_next_actions_mask"].float(), temperature)
    reward_loss = F.mse_loss(O.mlp(st.reward, batch["state"]).gather(1, idx), mrc)
    metric_q = O.mlp(st.qcpe, batch["state"]).gather(1, idx)
    with torch.no_grad():
        chunks = torch.chunk(O.mlp(st.qcpe_t, batch["next_state"]), M, dim=1)
        tgt = torch.cat([mrc[:, i:i + 1] + gamma * (c * prop).sum(1, keepdim=True)
                         * batch["not_terminal"] for i, c in enumerate(chunks)], dim=1)
    fn = F.mse_loss if loss == "mse" else F.smooth_l1_loss
    return reward_loss, fn(metric_q, tgt)


# ---------------------------------------------------------------------------
# compact goldens: networks too large to store (the CartPole configuration's [1024, 1024])
# ---------------------------------------------------------------------------
def seeded_like(params, seed: int):
    """Reproducible initial values for a list of parameter tensors: weights N(0, 1/sqrt(fan_in)),
    biases N(0, 0.1), from one CPU generator."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for p in params:
        std = 0.1 if p.dim() == 1 else 1.0 / (p.shape[1] ** 0.5)
        out.append(torch.randn(p.shape, generator=gen) * std)
    return out


def digest(t: torch.Tensor, limit: int = 2048):
    """A strided sample of a tensor (at most ~`limit` elements) followed by its sum and the sum
    of its absolute values, in float64."""
    f = t.detach().double().cpu().reshape(-1)
    stride = max(1, -(-f.numel() // limit))
    return torch.cat([f[::stride], f.sum().view(1), f.abs().sum().view(1)])
