"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch fp32 + autograd) of the SACTrainer update
with a state-value network and optional CRR weighting of the actor loss
(reagent/training/sac_trainer.py:23-48, :109-113, :148-193, :214-343).  Never imported by the
product path.

PINNED: tests/test_sac_value_cpu.py checks it against the golden vectors that
oracle/make_sac_value_golden.py produced by running the UNMODIFIED reference SACTrainer.

`sample_weight` gives the prioritized-replay variant: each critic loss becomes
mean_b(w_b * (q_b - y_b)^2); the actor, alpha and value losses stay unweighted.
"""
import math
from typing import Optional

import torch
import torch.nn.functional as F

from oracle.td_oracle import (LOG_PROB_MAX, LOG_PROB_MIN, AdamState, _grad_step, clone_net,
                              critic, gaussian_actor_forward, mlp, net_params, soft_update)


def crr_weight(advantage, *, indicator_fn_threshold=None, exponent_beta=None,
               exponent_clamp=None):
    """CRRWeightFn.get_weight_from_advantage (sac_trainer.py:38-48)."""
    if indicator_fn_threshold:
        return (advantage >= indicator_fn_threshold).float()
    exp = torch.exp(advantage / exponent_beta)
    if exponent_clamp:
        exp = torch.clamp(exp, 0.0, exponent_clamp)
    return exp


class SacValueState:
    """Mutable state of the restated SACTrainer with a value network: no q targets, a value
    target copied from the value network (sac_trainer.py:109-113)."""

    def __init__(self, actor, q1, q2, value, *, lr=1e-3, entropy_temperature=0.01,
                 learn_alpha=True, target_entropy=-1.0, logged_action_uniform_prior=True,
                 crr: Optional[dict] = None):
        self.actor, self.q1, self.q2, self.value = actor, q1, q2, value
        self.value_t = clone_net(value)
        for n in (actor, q1, q2, value):
            if n is not None:
                for p in net_params(n):
                    p.requires_grad_(True)
        self.alpha = entropy_temperature
        self.learn_alpha = learn_alpha
        self.target_entropy = target_entropy
        self.uniform_prior = logged_action_uniform_prior
        self.crr = crr
        self.adam_q1 = AdamState(net_params(q1), lr=lr)
        self.adam_q2 = None if q2 is None else AdamState(net_params(q2), lr=lr)
        self.adam_actor = AdamState(net_params(actor), lr=lr)
        self.adam_value = AdamState(net_params(value), lr=lr)
        if learn_alpha:
            # float64, as torch.tensor([np.log(x)]) is in the reference (sac_trainer.py:122-126)
            self.log_alpha = torch.tensor([math.log(entropy_temperature)], dtype=torch.float64,
                                          requires_grad=True)
            self.adam_alpha = AdamState([self.log_alpha], lr=lr)


def _critic_loss(q, target, sample_weight):
    if sample_weight is None:
        return F.mse_loss(q, target)
    return (sample_weight.reshape(-1, 1) * (q - target) ** 2).mean()


def sac_value_update(st: SacValueState, batch, noise_cur, *, gamma, tau,
                     sample_weight: Optional[torch.Tensor] = None):
    """One update.  Returns dict(losses=[q1, (q2), actor, (alpha), value], grads={...},
    target=[B, 1] TD target, td_error=[B] max_c |q_c - y|)."""
    state, action = batch["state"], batch["action"]
    reward, not_done = batch["reward"], batch["not_terminal"].float()
    # --- target (:214-217, :233-239): V'(s'), no actor forward on s' ---
    next_v = mlp(st.value_t, batch["next_state"])
    discount = torch.full_like(reward, gamma)
    target = (reward + discount * next_v * not_done) if gamma > 0.0 else reward
    target = target.detach()
    out = {"losses": [], "grads": {}, "target": target}
    # --- critics (:241-248) ---
    q1v = critic(st.q1, state, action)
    td = (q1v - target).abs().reshape(-1).detach()
    q1_loss = _critic_loss(q1v, target, sample_weight)
    out["grads"]["q1"] = _grad_step(q1_loss, st.q1, st.adam_q1)
    out["losses"].append(float(q1_loss))
    if st.q2 is not None:
        q2v = critic(st.q2, state, action)
        td = torch.maximum(td, (q2v - target).abs().reshape(-1).detach())
        q2_loss = _critic_loss(q2v, target, sample_weight)
        out["grads"]["q2"] = _grad_step(q2_loss, st.q2, st.adam_q2)
        out["losses"].append(float(q2_loss))
    out["td_error"] = td
    # --- actor (:254-283), sees the updated critics ---
    a_cur, logp = gaussian_actor_forward(st.actor, state, noise_cur)
    min_q = critic(st.q1, state, a_cur)
    if st.q2 is not None:
        min_q = torch.min(min_q, critic(st.q2, state, a_cur))
    actor_log_prob = logp.clamp(LOG_PROB_MIN, LOG_PROB_MAX)
    if st.crr is not None:
        advantage = (min_q - mlp(st.value, state)).detach()
        w = crr_weight(advantage, **st.crr)
        actor_loss = (-(actor_log_prob * w.detach())).mean()
    else:
        actor_loss = (st.alpha * actor_log_prob - min_q).mean()
    out["grads"]["actor"] = _grad_step(actor_loss, st.actor, st.adam_actor)
    out["losses"].append(float(actor_loss))
    # --- alpha (:311-322) ---
    if st.learn_alpha:
        alpha_loss = -(
            (st.log_alpha * (logp.clamp(LOG_PROB_MIN, LOG_PROB_MAX) + st.target_entropy).detach())
            .mean())
        out["grads"]["alpha"] = _grad_step(alpha_loss, [st.log_alpha], st.adam_alpha)
        out["losses"].append(float(alpha_loss))
        st.alpha = st.log_alpha.detach().exp()
    # --- value (:329-343), with the post-update alpha ---
    if st.uniform_prior:
        target_value = min_q
    else:
        target_value = min_q - st.alpha * logp.clamp(LOG_PROB_MIN, LOG_PROB_MAX)
    state_value = mlp(st.value, state)
    value_loss = F.mse_loss(state_value, target_value.detach().to(state_value.dtype))
    out["grads"]["value"] = _grad_step(value_loss, st.value, st.adam_value)
    out["losses"].append(float(value_loss))
    # --- soft update of the value target only (:176-193) ---
    soft_update(st.value_t, st.value, tau)
    return out
