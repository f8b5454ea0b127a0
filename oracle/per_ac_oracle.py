"""Prioritized replay for SAC and TD3, on top of td_oracle: the importance-weighted critic
updates and the twin-critic priorities that FusedPolicyStep(per=PrioritizedUpdate(...)) computes
on the GPU for SACTrainer and TD3Trainer.

The updates restate td_oracle.sac_update / td3_update with each critic's F.mse_loss replaced by
mean_b(w_b * (q_b - y_b)^2); with w = 1 they reduce to those updates, which are pinned to the
reference's goldens.  The actor and alpha losses stay unweighted: the importance weights correct
the bias of the critics' regression towards the sampled TD targets (Schaul et al. 2016).  A
row's priority is the larger of the two critics' absolute TD errors, the convention of the PER
baselines for TD3 in Fujimoto, Meger & Precup 2020."""
import numpy as np
import torch

from . import td_oracle as O


def _weighted_mse(q, target, weights):
    d = q - target
    if weights is None:
        return torch.mean(d * d), d
    return torch.mean(weights.reshape(-1, 1) * (d * d)), d


def _critics(st, state, action, target, weights, out):
    """Weighted critic losses and Adam steps of q1 (and q2); returns [B] max_c |q_c - y|."""
    q1 = O.critic(st.q1, state, action)
    q1_loss, d1 = _weighted_mse(q1, target, weights)
    out["q1_value"] = q1.detach().reshape(-1)
    out["grads"]["q1"] = O._grad_step(q1_loss, st.q1, st.adam_q1)
    out["losses"].append(float(q1_loss.detach()))
    td_error = d1.detach().abs().reshape(-1)
    if st.q2 is not None:
        q2 = O.critic(st.q2, state, action)
        q2_loss, d2 = _weighted_mse(q2, target, weights)
        out["q2_value"] = q2.detach().reshape(-1)
        out["grads"]["q2"] = O._grad_step(q2_loss, st.q2, st.adam_q2)
        out["losses"].append(float(q2_loss.detach()))
        td_error = torch.maximum(td_error, d2.detach().abs().reshape(-1))
    out["td_error"] = td_error
    return td_error


def weighted_sac_update(st: O.SacState, batch, noise_next, noise_cur, weights, *, gamma, tau,
                        backprop_through_log_prob=True):
    """td_oracle.sac_update with importance-weighted critic losses (`weights` [B] or None).
    Returns dict(losses, grads, target, q1_value, q2_value, td_error)."""
    state, action = batch["state"], batch["action"]
    reward, not_done = batch["reward"], batch["not_terminal"].float()
    a_next, _ = O.gaussian_actor_forward(st.actor, batch["next_state"], noise_next)
    next_v = O.critic(st.q1t, batch["next_state"], a_next)
    if st.q2 is not None:
        next_v = torch.min(next_v, O.critic(st.q2t, batch["next_state"], a_next))
    log_prob_a = O.gaussian_log_prob(st.actor, batch["next_state"], a_next).clamp(
        O.LOG_PROB_MIN, O.LOG_PROB_MAX)
    next_v = (next_v - st.alpha * log_prob_a).float()
    discount = torch.full_like(reward, gamma)
    target = (reward + discount * next_v * not_done) if gamma > 0.0 else reward
    target = target.detach()
    out = {"losses": [], "grads": {}, "target": target}
    _critics(st, state, action, target, weights, out)
    # actor and alpha: unweighted, as td_oracle.sac_update
    a_cur, logp = O.gaussian_actor_forward(st.actor, state, noise_cur)
    min_q = O.critic(st.q1, state, a_cur)
    if st.q2 is not None:
        min_q = torch.min(min_q, O.critic(st.q2, state, a_cur))
    actor_log_prob = logp.clamp(O.LOG_PROB_MIN, O.LOG_PROB_MAX)
    if not backprop_through_log_prob:
        actor_log_prob = actor_log_prob.detach()
    actor_loss = (st.alpha * actor_log_prob - min_q).mean()
    out["grads"]["actor"] = O._grad_step(actor_loss, st.actor, st.adam_actor)
    out["losses"].append(float(actor_loss.detach()))
    if st.learn_alpha:
        alpha_loss = -(
            (st.log_alpha * (logp.clamp(O.LOG_PROB_MIN, O.LOG_PROB_MAX) + st.target_entropy)
             .detach()).mean())
        out["grads"]["alpha"] = O._grad_step(alpha_loss, [st.log_alpha], st.adam_alpha)
        out["losses"].append(float(alpha_loss.detach()))
        st.alpha = st.log_alpha.detach().exp()
    O.soft_update(st.q1t, st.q1, tau)
    if st.q2 is not None:
        O.soft_update(st.q2t, st.q2, tau)
    return out


def weighted_td3_update(st: O.Td3State, batch, noise_next, batch_idx, weights, *, gamma, tau,
                        noise_variance=0.2, noise_clip=0.5, delayed_policy_update=2):
    """td_oracle.td3_update with importance-weighted critic losses (`weights` [B] or None)."""
    state, action = batch["state"], batch["action"]
    with torch.no_grad():
        next_actor = O.mlp(st.actor_t, batch["next_state"])
        noise = noise_next * noise_variance
        next_actor = (next_actor + noise.clamp(-noise_clip, noise_clip)).clamp(-1.0, 1.0)
        next_q = O.critic(st.q1t, batch["next_state"], next_actor)
        if st.q2 is not None:
            next_q = torch.min(next_q, O.critic(st.q2t, batch["next_state"], next_actor))
        target = batch["reward"] + gamma * next_q * batch["not_terminal"].float()
    out = {"losses": [], "grads": {}, "target": target}
    _critics(st, state, action, target, weights, out)
    if batch_idx % delayed_policy_update == 0:
        actor_loss = -(O.critic(st.q1, state, O.mlp(st.actor, state)).mean())
        out["grads"]["actor"] = O._grad_step(actor_loss, st.actor, st.adam_actor)
        out["losses"].append(float(actor_loss.detach()))
        O.soft_update(st.q1t, st.q1, tau)
        if st.q2 is not None:
            O.soft_update(st.q2t, st.q2, tau)
        O.soft_update(st.actor_t, st.actor, tau)
    else:
        out["losses"].append(None)
    return out


def twin_td_priorities(q1_value, q2_value, td_target, alpha, eps):
    """p_b = ((double)max(|q1_b - y_b|, |q2_b - y_b|) + eps) ** alpha in fp64, the differences
    taken in fp32 (q2_value None: one critic)."""
    q1 = np.asarray(q1_value, np.float32)
    y = np.asarray(td_target, np.float32)
    e = np.abs(q1 - y)
    if q2_value is not None:
        e = np.maximum(e, np.abs(np.asarray(q2_value, np.float32) - y))
    return (e.astype(np.float64) + eps) ** alpha
