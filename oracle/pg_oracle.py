"""Plain-torch restatement of ReinforceTrainer.train_step_gen (reagent/training/
reinforce_trainer.py:92-148) and PPOTrainer._update_model (reagent/training/ppo_trainer.py:
271-444, 540-563), plus fp64 references of the two kernels of rb200_pg.cu.

Networks are td_oracle dicts (plain or dueling); the policy's scores are masked with
INVALID_ACTION_CONSTANT like FullyConnectedDQN.forward, then divided by the sampler's
temperature (SoftmaxActionSampler._get_distribution)."""
import math
from typing import Dict, List

import numpy as np
import torch

from oracle import td_oracle as O

EPS = np.finfo(float).eps.item()
INVALID_ACTION_CONSTANT = -1e10


def discounted_returns(rewards: torch.Tensor, gamma: float = 0) -> torch.Tensor:
    """utils.py:42-54: the fp32 loop of 0-dim tensor ops (what rb200_pg_returns reproduces)."""
    if gamma == 0:
        return rewards.float()
    returns = torch.empty_like(rewards, dtype=torch.float)
    running = torch.zeros((), dtype=torch.float, device=rewards.device)
    for t in range(rewards.shape[0] - 1, -1, -1):
        running = rewards[t].float() + gamma * running
        returns[t] = running
    return returns


def whiten(x: torch.Tensor, subtract_mean: bool) -> torch.Tensor:
    """utils.py:32-39: population std + EPS."""
    std = x.std(unbiased=False)
    numer = x - x.mean() if subtract_mean else x
    return numer / (std + EPS)


def logits(scores, mask, temperature):
    if mask is not None:
        scores = scores + INVALID_ACTION_CONSTANT * (1 - mask.float())
    return scores / temperature


def log_prob(scores, mask, action, temperature):
    """SoftmaxActionSampler.log_prob: Categorical(logits).log_prob(action.argmax(1))."""
    d = torch.distributions.Categorical(logits=logits(scores, mask, temperature))
    return d.log_prob(action.argmax(dim=1))


def entropy(scores, mask, temperature):
    return torch.distributions.Categorical(logits=logits(scores, mask, temperature)).entropy().mean()


def _grads(loss, params):
    return list(torch.autograd.grad(loss, params, allow_unused=True))


def reinforce_update(policy, value, adam_p, adam_v, traj: Dict[str, torch.Tensor], *, gamma,
                     off_policy, reward_clip, clip_param, normalize, subtract_mean,
                     offset_clamp_min, temperature):
    """One update.  Returns (losses [value?, policy], grads [value?, policy], returns,
    advantage)."""
    scores = O.mlp(policy, traj["state"])
    elig = log_prob(scores, traj.get("possible_actions_mask"), traj["action"], temperature).float()
    ret = discounted_returns(torch.clamp(traj["reward"], max=reward_clip).clone(), gamma)
    adv = ret
    if normalize:
        adv = whiten(adv, subtract_mean=subtract_mean)
    elif subtract_mean:
        adv = adv - adv.mean()
    if offset_clamp_min:
        adv = adv.clamp(min=0)
    losses, grads = [], []
    if value is not None:
        base = O.mlp(value, traj["state"]).squeeze()
        vloss = torch.nn.functional.mse_loss(base, adv)
        losses.append(float(vloss))
        grads.append(_grads(vloss, O.net_params(value)))
        adv = adv - base.detach()
    if off_policy:
        elig = torch.exp(torch.clamp(elig - traj["log_prob"], max=math.log(float(clip_param))))
    loss = -(adv.float().detach()) @ elig
    losses.append(float(loss))
    grads.append(_grads(loss, O.net_params(policy)))
    if value is not None:
        adam_v.step(O.net_params(value), grads[0])
    adam_p.step(O.net_params(policy), grads[-1])
    return losses, grads, ret.detach(), adv.detach().reshape(-1)


def ppo_advantage(value, traj, *, gamma, reward_clip, normalize, subtract_mean,
                  offset_clamp_min, td_error_advantage):
    """PPOTrainer._compute_advantage / _td_error_advantage: (advantage, value loss or None)."""
    rewards = traj["reward"]
    if value is not None and td_error_advantage:
        base = O.mlp(value, traj["state"]).reshape(-1)
        v = base.detach()
        r = torch.clamp(rewards, max=reward_clip).reshape(-1)
        nt = traj.get("not_terminal")
        if nt is None:
            nt = torch.ones_like(v)
            nt[-1] = 0.0
        if traj.get("next_state") is not None:
            nv = O.mlp(value, traj["next_state"]).detach().reshape(-1)
        else:
            nv = torch.cat([v[1:], v.new_zeros(1)])
        y = r + gamma * nt * nv
        vloss = torch.nn.functional.mse_loss(base, y, reduction="sum")
        adv = y - v
        if offset_clamp_min:
            adv = adv.clamp(min=0)
        return adv, vloss
    adv = discounted_returns(torch.clamp(rewards, max=reward_clip).clone(), gamma)
    if normalize:
        adv = whiten(adv, subtract_mean=subtract_mean)
    if offset_clamp_min:
        adv = adv.clamp(min=0)
    vloss = None
    if value is not None:
        base = O.mlp(value, traj["state"]).squeeze().reshape(-1)
        vloss = torch.nn.functional.mse_loss(base, adv, reduction="sum")
        adv = adv - base.detach()
    return adv, vloss


def ppo_update(policy, value, adam_p, adam_v, trajs: List[Dict[str, torch.Tensor]], *, gamma,
               reward_clip, normalize, subtract_mean, offset_clamp_min, td_error_advantage,
               ppo_epsilon, entropy_weight, temperature):
    """One _update_model over a minibatch.  Returns (losses [value?, ppo], grads [value?, ppo],
    advantages of the packed rows)."""
    ppo, vl, advs = [], [], []
    for t in trajs:
        adv, vloss = ppo_advantage(value, t, gamma=gamma, reward_clip=reward_clip,
                                   normalize=normalize, subtract_mean=subtract_mean,
                                   offset_clamp_min=offset_clamp_min,
                                   td_error_advantage=td_error_advantage)
        if vloss is not None:
            vl.append(vloss)
        scores = O.mlp(policy, t["state"])
        mask = t.get("possible_actions_mask")
        lp = log_prob(scores, mask, t["action"], temperature).float()
        rho = torch.exp(lp - t["log_prob"].detach()).float()
        adv = adv.float().detach()
        surr = torch.min(adv * rho, adv * torch.clamp(rho, 1 - ppo_epsilon, 1 + ppo_epsilon))
        loss = -surr.sum()
        if entropy_weight != 0:
            loss = loss - entropy_weight * (entropy(scores, mask, temperature) * scores.shape[0])
        ppo.append(loss)
        advs.append(adv)
    losses, grads = [], []
    if value is not None:
        v = torch.stack(vl).sum()
        losses.append(float(v))
        grads.append(_grads(v, O.net_params(value)))
    p = torch.stack(ppo).sum()
    losses.append(float(p))
    grads.append(_grads(p, O.net_params(policy)))
    if value is not None:
        adam_v.step(O.net_params(value), grads[0])
    adam_p.step(O.net_params(policy), grads[-1])
    return losses, grads, torch.cat(advs)


# ---------------------------------------------------------------------------
# fp64 references of the kernels
# ---------------------------------------------------------------------------
def returns_fp64(reward, offsets, *, gamma, reward_clip, normalize, subtract_mean,
                 offset_clamp_min, ppo=False):
    """rb200_pg_returns in fp64 (ppo: no mean subtraction without normalize)."""
    out = []
    r = torch.as_tensor(reward, dtype=torch.float64)
    for i in range(len(offsets) - 1):
        x = torch.clamp(r[offsets[i]:offsets[i + 1]], max=reward_clip)
        if gamma != 0:
            run, y = 0.0, torch.empty_like(x)
            for t in range(len(x) - 1, -1, -1):
                run = float(x[t]) + gamma * run
                y[t] = run
            x = y
        if normalize:
            m = x.mean()
            x = ((x - m) if subtract_mean else x) / (x.std(unbiased=False) + EPS)
        elif subtract_mean and not ppo:
            x = x - x.mean()
        if offset_clamp_min:
            x = x.clamp(min=0)
        out.append(x)
    return torch.cat(out)


def head_fp64(scores, mask, action, advantage, *, temperature, ppo, logged=None,
              clip_param=None, ppo_epsilon=0.2, entropy_weight=0.0):
    """rb200_pg_head's policy part in fp64 given the advantage: (policy loss, d loss / d
    scores)."""
    z = torch.as_tensor(scores, dtype=torch.float64).clone().requires_grad_(True)
    m = None if mask is None else torch.as_tensor(mask, dtype=torch.float64)
    a = torch.as_tensor(action, dtype=torch.float64)
    adv = torch.as_tensor(advantage, dtype=torch.float64)
    lg = logits(z, m, temperature)
    lp = torch.log_softmax(lg, 1).gather(1, a.argmax(1, keepdim=True)).squeeze(1)
    if ppo:
        rho = torch.exp(lp - torch.as_tensor(logged, dtype=torch.float64))
        loss = -torch.min(adv * rho, adv * torch.clamp(rho, 1 - ppo_epsilon, 1 + ppo_epsilon)).sum()
        if entropy_weight != 0:
            p = torch.softmax(lg, 1)
            loss = loss - entropy_weight * (-(p * torch.log_softmax(lg, 1)).sum())
    else:
        elig = lp
        if logged is not None:
            elig = torch.exp(torch.clamp(lp - torch.as_tensor(logged, dtype=torch.float64),
                                         max=math.log(clip_param)))
        loss = -(adv @ elig)
    loss.backward()
    return float(loss), z.grad


def pack_offsets(lengths: List[int]) -> List[int]:
    offs = [0]
    for n in lengths:
        offs.append(offs[-1] + n)
    return offs
