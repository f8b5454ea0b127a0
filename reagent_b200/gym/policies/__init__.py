"""Act-time side of the path (SURVEY.md 8f rank 2): scores from the fused Q-network forward,
then an action sampler -- the reference's Policy = scorer o sampler composition.

  discrete_dqn_scorer        reagent/gym/policies/scorers/discrete_scorer.py:16-48
  parametric_dqn_scorer      reagent/gym/policies/scorers/discrete_scorer.py:65-87
  slate_q_scorer, TopKSampler
                             reagent/gym/policies/scorers/slate_q_scorer.py:13-30,
                             reagent/gym/policies/samplers/top_k_sampler.py
  Greedy / EpsilonGreedy / Softmax samplers
                             reagent/gym/policies/samplers/discrete_sampler.py:14-183
  Policy                     reagent/gym/policies/policy.py:13-43
  ActorPolicyWrapper         reagent/model_managers/actor_critic_base.py:51-64 (continuous actors)

The scorer runs `q_network(obs)` (ONE fused launch, rb200_mlp_forward; a QR-DQN head is
averaged over atoms) on the GPU -- for a parametric q network, q(obs, a) of every one-hot action
a in one rb200_mlp_forward_tiled launch; the samplers are index / probability arithmetic on the (B, A)
score tensor with torch's own RNG, so a seeded draw reproduces the reference's draw.
"""
from typing import Any, Optional

import torch
import torch.nn.functional as F

from ...core import types as rlt
from ...models.dqn import INVALID_ACTION_CONSTANT

NEG_INF = float("-inf")


def apply_possible_actions_mask(scores: torch.Tensor,
                                possible_actions_mask: Optional[torch.Tensor] = None,
                                invalid_score: float = NEG_INF) -> torch.Tensor:
    """Overwrite the scores of impossible actions (mask is for ONE observation: (A,) bool)."""
    if possible_actions_mask is None:
        return scores
    mask = possible_actions_mask.unsqueeze(0).to(scores.device)
    assert scores.shape == mask.shape, f"{scores.shape} != {mask.shape}"
    scores[~mask] = invalid_score
    return scores


def discrete_dqn_scorer(q_network):
    @torch.no_grad()
    def score(preprocessed_obs: rlt.FeatureData,
              possible_actions_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        was_training = q_network.training
        q_network.eval()
        scores = q_network(preprocessed_obs)
        if scores.dim() == 3:  # QR-DQN: (batch, actions, atoms) -> expected value
            scores = scores.mean(dim=2)
        assert scores.dim() == 2, f"{scores.shape} isn't (batchsize, num_actions)."
        q_network.train(was_training or True)  # the reference always switches back to train()
        return apply_possible_actions_mask(scores, possible_actions_mask)

    return score


def parametric_dqn_scorer(max_num_actions: int, q_network):
    """Scores (n, max_num_actions) of q_network(obs[i], e_a) for every one-hot action e_a, the
    reference's get_parametric_input (obs.get_tiled_batch + get_possible_actions_for_gym).  The
    repeated observations are built per row tile inside the forward kernel and never exist in
    memory; the (n * max_num_actions, max_num_actions) identity tiling is a device tensor,
    cached for the last n."""
    from ...models.arena import run_mlp_tiled

    eyes = {}

    @torch.no_grad()
    def score(preprocessed_obs: rlt.FeatureData) -> torch.Tensor:
        obs = preprocessed_obs.float_features
        assert obs.dim() == 2, f"{obs.shape} is not (batch_size, state_dim)."
        arena = q_network.arena
        dev = arena.flat.device
        obs = obs.to(dev, torch.float32).contiguous()
        n = obs.shape[0]
        key = (n, str(dev))
        if key not in eyes:
            eyes.clear()
            eyes[key] = torch.eye(max_num_actions, device=dev).repeat(n, 1)
        q_network.eval()
        out = torch.empty(n * max_num_actions, arena.dims[-1], device=dev)
        run_mlp_tiled([arena], obs, eyes[key], max_num_actions, [out])
        q_network.train()
        return out.view(-1, max_num_actions)

    return score


def slate_q_scorer(num_candidates: int, q_network):
    """reagent/gym/policies/scorers/slate_q_scorer.py:13-30: softmax(candidate value) times
    q_network(state, candidate) for every candidate of every row, (n, num_candidates).  The
    repeated states are built per row tile inside one rb200_mlp_forward_tiled launch."""
    from ...models.arena import run_mlp_tiled

    @torch.no_grad()
    def score(state: rlt.FeatureData) -> torch.Tensor:
        docs = state.candidate_docs
        assert docs is not None
        arena = q_network.arena
        dev = arena.flat.device
        obs = state.float_features.to(dev, torch.float32).contiguous()
        n = obs.shape[0]
        cand = docs.float_features.to(dev, torch.float32).reshape(n * num_candidates, -1).contiguous()
        q_network.eval()
        out = torch.empty(n * num_candidates, arena.dims[-1], device=dev)
        run_mlp_tiled([arena], obs, cand, num_candidates, [out])
        q_network.train()
        scores = out.view(-1, num_candidates)
        select_prob = F.softmax(docs.value.to(dev), dim=1)
        assert select_prob.shape == scores.shape
        return select_prob * scores

    return score


class TopKSampler:
    """reagent/gym/policies/samplers/top_k_sampler.py: the indices of the k best scores of each
    row, log_prob 0."""

    def __init__(self, k: int) -> None:
        self.k = k

    def sample_action(self, scores: torch.Tensor) -> rlt.ActorOutput:
        _, item_idxs = torch.topk(scores, self.k, dim=1)
        return rlt.ActorOutput(action=item_idxs,
                               log_prob=torch.zeros(item_idxs.shape[0], 1, device=scores.device))

    def log_prob(self, scores: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError


class GreedyActionSampler:
    """arg max of the scores; log_prob 0."""

    @torch.no_grad()
    def sample_action(self, scores: torch.Tensor) -> rlt.ActorOutput:
        assert scores.dim() == 2, f"scores shape is {scores.shape}, not (batchsize, num_actions)"
        idx = scores.argmax(dim=1)
        return rlt.ActorOutput(action=F.one_hot(idx, scores.shape[1]),
                               log_prob=torch.zeros_like(idx, dtype=torch.float))

    @torch.no_grad()
    def log_prob(self, scores: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
        # discrete_sampler.py:111-117 as written upstream: -inf where the action IS the greedy one
        hit = scores.argmax(dim=1) == action.argmax(-1)
        lp = torch.zeros(scores.shape[0], device=scores.device).float()
        lp[hit] = -float("inf")
        return lp


class EpsilonGreedyActionSampler:
    """With probability epsilon a uniformly random VALID action (score > INVALID_ACTION_CONSTANT),
    else the greedy one; update() decays epsilon."""

    def __init__(self, epsilon: float, epsilon_decay: float = 1.0,
                 minimum_epsilon: float = 0.0) -> None:
        self.epsilon = float(epsilon)
        assert epsilon_decay <= 1
        self.epsilon_decay = epsilon_decay
        assert minimum_epsilon <= epsilon_decay
        self.minimum_epsilon = minimum_epsilon

    def action_probabilities(self, scores: torch.Tensor) -> torch.Tensor:
        assert scores.dim() == 2, "scores dim is %d" % scores.dim()
        n_actions = scores.shape[1]
        greedy = F.one_hot(scores.argmax(dim=1), n_actions).bool()
        valid = scores > INVALID_ACTION_CONSTANT
        explore = self.epsilon / valid.float().sum(1, keepdim=True)
        p = torch.zeros_like(scores) + explore
        p[greedy] = (1 - self.epsilon + explore).squeeze()
        p[~valid] = 0.0
        total = p.sum(1)
        assert torch.allclose(total, torch.ones_like(total))
        return p

    def sample_action(self, scores: torch.Tensor) -> rlt.ActorOutput:
        dist = torch.distributions.Categorical(probs=self.action_probabilities(scores))
        idx = dist.sample()
        return rlt.ActorOutput(action=F.one_hot(idx, scores.shape[1]), log_prob=dist.log_prob(idx))

    def log_prob(self, scores: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
        """discrete_sampler.py:166-172 as it BEHAVES upstream: it first draws an action (the RNG
        is consumed), then compares the drawn rlt.ActorOutput -- not its action tensor -- with
        `action.argmax(-1)`; that comparison is never true, so every entry is epsilon / n
        (pinned by the golden vector `eps.lp_of_action`)."""
        self.sample_action(scores)
        n = len(scores)
        return torch.ones(n, device=scores.device) * self.epsilon / n

    def update(self) -> None:
        self.epsilon *= self.epsilon_decay
        if self.minimum_epsilon is not None:
            self.epsilon = max(self.epsilon, self.minimum_epsilon)


class SoftmaxActionSampler:
    """Categorical over softmax(scores / temperature); update() decays the temperature."""

    def __init__(self, temperature: float = 1.0, temperature_decay: float = 1.0,
                 minimum_temperature: float = 0.1) -> None:
        assert temperature > 0, f"Invalid non-positive temperature {temperature}."
        assert temperature_decay <= 1.0, f"Invalid temperature_decay>1: {temperature_decay}."
        assert minimum_temperature <= temperature, (
            f"minimum_temperature ({minimum_temperature}) exceeds initial temperature ({temperature})")
        self.temperature = temperature
        self.temperature_decay = temperature_decay
        self.minimum_temperature = minimum_temperature

    def _dist(self, scores: torch.Tensor) -> torch.distributions.Categorical:
        return torch.distributions.Categorical(logits=scores / self.temperature)

    @torch.no_grad()
    def sample_action(self, scores: torch.Tensor) -> rlt.ActorOutput:
        assert scores.dim() == 2, f"scores shape is {scores.shape}, not (batch_size, num_actions)"
        dist = self._dist(scores)
        idx = dist.sample()
        assert idx.shape == (scores.shape[0],)
        return rlt.ActorOutput(action=F.one_hot(idx, scores.shape[1]), log_prob=dist.log_prob(idx))

    def log_prob(self, scores: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
        assert scores.dim() == 2 and scores.shape == action.shape, f"{scores.shape} != {action.shape}"
        return self._dist(scores).log_prob(action.argmax(dim=1))

    def entropy(self, scores: torch.Tensor) -> torch.Tensor:
        assert scores.dim() == 2, f"{scores.shape}"
        return self._dist(scores).entropy().mean()

    def update(self) -> None:
        self.temperature = max(self.temperature * self.temperature_decay, self.minimum_temperature)


class Policy:
    """scores = scorer(obs[, mask]); action = sampler.sample_action(scores), returned on the CPU
    (these are the actions that go into the replay buffer)."""

    def __init__(self, scorer, sampler) -> None:
        self.scorer = scorer
        self.sampler = sampler

    def act(self, obs: Any, possible_actions_mask: Optional[torch.Tensor] = None) -> rlt.ActorOutput:
        args = (obs,) if possible_actions_mask is None else (obs, possible_actions_mask)
        out = self.sampler.sample_action(self.scorer(*args))
        return out.cpu().detach()


class ActorPolicyWrapper(Policy):
    """Continuous control: the actor network IS the policy (its forward samples the action)."""

    def __init__(self, actor_network):
        self.actor_network = actor_network

    @torch.no_grad()
    def act(self, obs: rlt.FeatureData, possible_actions_mask: Optional[torch.Tensor] = None) -> rlt.ActorOutput:
        self.actor_network.eval()
        out = self.actor_network(obs)
        self.actor_network.train()
        return out.detach().cpu()
