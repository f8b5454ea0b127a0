"""Replay batch -> trainer batch makers with the reference's call contract
(reagent/gym/preprocessors/trainer_preprocessor.py:32-227).  These operate on a replay
namedtuple that is already on the GPU (a few elementwise torch ops on (B, A) tensors); the
hot path uses ReplayBuffer.sample_discrete_dqn_batch / sample_policy_network_batch, which
produce the same batches inside the fused sample kernel."""
import inspect
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from ...core import types as rlt
from ...core.parameters import CONTINUOUS_TRAINING_ACTION_RANGE


def rescale_actions(actions, new_min, new_max, prev_min, prev_max):
    """reagent/training/utils.py:13-29"""
    prev_range = prev_max - prev_min
    new_range = new_max - new_min
    return ((actions - prev_min) / prev_range) * new_range + new_min


def one_hot_actions(num_actions, action, next_action, terminal):
    """trainer_preprocessor.py:72-97"""
    assert len(action.shape) == 2 and action.shape[1] == 1 and next_action.shape == action.shape
    action = F.one_hot(action, num_actions).squeeze(1).float()
    next_action_res = torch.zeros_like(action)
    non_terminal_indices = (terminal == 0).squeeze(1)
    next_action_res[non_terminal_indices] = (
        F.one_hot(next_action[non_terminal_indices], num_actions).squeeze(1).float())
    return action, next_action_res


class DiscreteDqnInputMaker:
    def __init__(self, num_actions: int, trainer_preprocessor=None):
        self.num_actions = num_actions
        self.trainer_preprocessor = trainer_preprocessor

    @classmethod
    def create_for_env(cls, env):
        return cls(num_actions=env.action_space.n,
                   trainer_preprocessor=getattr(env, "trainer_preprocessor", None))

    def __call__(self, batch):
        not_terminal = 1.0 - batch.terminal.float()
        action, next_action = one_hot_actions(self.num_actions, batch.action, batch.next_action,
                                              batch.terminal)
        if self.trainer_preprocessor is not None:
            state = self.trainer_preprocessor(batch.state)
            next_state = self.trainer_preprocessor(batch.next_state)
        else:
            state = rlt.FeatureData(float_features=batch.state)
            next_state = rlt.FeatureData(float_features=batch.next_state)
        pam = getattr(batch, "possible_actions_mask", None)
        pnam = getattr(batch, "next_possible_actions_mask", None)
        possible_actions_mask = pam.float() if pam is not None else torch.ones_like(action)
        possible_next_actions_mask = pnam.float() if pnam is not None else torch.ones_like(next_action)
        log_prob = getattr(batch, "log_prob", None)
        return rlt.DiscreteDqnInput(
            state=state, action=action, next_state=next_state, next_action=next_action,
            possible_actions_mask=possible_actions_mask,
            possible_next_actions_mask=possible_next_actions_mask, reward=batch.reward,
            not_terminal=not_terminal, step=None, time_diff=None,
            extras=rlt.ExtraData(action_probability=None if log_prob is None else log_prob.exp()))


class PolicyNetworkInputMaker:
    def __init__(self, action_low: np.ndarray, action_high: np.ndarray):
        self.action_low = torch.tensor(action_low)
        self.action_high = torch.tensor(action_high)
        (train_low, train_high) = CONTINUOUS_TRAINING_ACTION_RANGE
        self.train_low = torch.tensor(train_low)
        self.train_high = torch.tensor(train_high)

    @classmethod
    def create_for_env(cls, env):
        return cls(env.action_space.low, env.action_space.high)

    def __call__(self, batch):
        dev = batch.action.device
        lo, hi = self.action_low.to(dev), self.action_high.to(dev)
        not_terminal = 1.0 - batch.terminal.float()
        action = rescale_actions(batch.action, self.train_low.to(dev), self.train_high.to(dev), lo, hi)
        non_terminal_indices = (batch.terminal == 0).squeeze(1)
        next_action = torch.zeros_like(action)
        next_action[non_terminal_indices] = rescale_actions(
            batch.next_action[non_terminal_indices], self.train_low.to(dev),
            self.train_high.to(dev), lo, hi)
        log_prob = getattr(batch, "log_prob", None)
        return rlt.PolicyNetworkInput(
            state=rlt.FeatureData(batch.state), next_state=rlt.FeatureData(batch.next_state),
            action=rlt.FeatureData(action), next_action=rlt.FeatureData(next_action),
            reward=batch.reward, not_terminal=not_terminal, step=None, time_diff=None,
            extras=rlt.ExtraData(action_probability=None if log_prob is None else log_prob.exp()))


class MemoryNetworkInputMaker:
    """trainer_preprocessor.py:281-354: a ReplayBuffer(stack_size=T,
    return_everything_as_stack=True) batch -> a time-major MemoryNetworkInput.  Layout only:
    one-hot discrete actions, [B, dim, T] -> [T, B, dim], [B, T] -> [T, B], and
    not_terminal = 1 before the last step of the stack."""

    def __init__(self, num_actions: Optional[int] = None):
        self.num_actions = num_actions

    @classmethod
    def create_for_env(cls, env):
        n = getattr(env.action_space, "n", None)
        if n is not None:
            return cls(int(n))
        if getattr(env.action_space, "low", None) is not None:
            return cls()
        raise NotImplementedError()

    def __call__(self, batch):
        action = batch.action
        if self.num_actions is not None:
            assert action.dim() == 2, f"{tuple(action.shape)}"
            # [B, T] indices -> [B, A, T]
            action = F.one_hot(action, self.num_actions).float().transpose(1, 2)

        def vector(name, t):  # [B, dim] (T == 1) or [B, dim, T] -> [T, B, dim]
            if t.dim() == 2:
                t = t.unsqueeze(2)
            assert t.dim() == 3, f"{name} has shape {tuple(t.shape)}"
            return t.permute(2, 0, 1)

        def scalar(name, t):  # [B] or [B, T] -> [T, B]
            if t.dim() == 1:
                t = t.unsqueeze(1)
            assert t.dim() == 2, f"{name} has shape {tuple(t.shape)}"
            return t.transpose(0, 1)

        reward = scalar("reward", batch.reward)
        not_terminal = scalar("not_terminal", 1.0 - batch.terminal.float())
        if reward.shape[0] > 1:
            # the replay buffer returns the terminal flag of the last step only: the earlier
            # steps of a stack cannot have been terminal
            assert not_terminal.shape == (1, reward.shape[1]), f"{tuple(not_terminal.shape)}"
            stacked = torch.ones_like(reward)
            stacked[-1] = not_terminal
            not_terminal = stacked
        return rlt.MemoryNetworkInput.from_dict({
            "state": vector("state", batch.state),
            "next_state": vector("next_state", batch.next_state),
            "action": vector("action", action),
            "reward": reward,
            "not_terminal": not_terminal,
            "step": None,
            "time_diff": None,
        })


class SlateQInputMaker:
    """trainer_preprocessor.py:230-278: a replay batch with the extras doc,
    augmentation_value, response_click and response_watch_time (and their next_ forms) -> a
    SlateQInput.  A null slot is appended to every slate: index slate_size in action /
    next_action, reward 0 in position_reward, and in reward_mask True exactly when nothing
    was clicked.  Every candidate is present (item masks of ones)."""

    def __init__(self):
        self.metric = "watch_time"

    @classmethod
    def create_for_env(cls, env):
        return cls()

    def __call__(self, batch):
        n = batch.state.shape[0]
        dev = batch.state.device
        item_mask = torch.ones(batch.doc.shape[:2], device=dev)
        next_item_mask = torch.ones(batch.doc.shape[:2], device=dev)
        null_action = torch.full((n, 1), batch.action.shape[1], dtype=torch.int64, device=dev)
        action = torch.cat([batch.action, null_action], dim=1)
        next_action = torch.cat([batch.next_action, null_action], dim=1)
        position_reward = getattr(batch, f"response_{self.metric}")
        position_reward = torch.cat([position_reward, torch.zeros((n, 1), device=dev)], dim=1)
        reward_mask = batch.response_click
        null_mask = (reward_mask.sum(dim=1) == 0).view(n, 1)
        reward_mask = torch.cat([reward_mask.to(torch.bool), null_mask], dim=1)
        return rlt.SlateQInput.from_dict({
            "state_features": batch.state,
            "next_state_features": batch.next_state,
            "candidate_features": batch.doc,
            "next_candidate_features": batch.next_doc,
            "item_mask": item_mask,
            "next_item_mask": next_item_mask,
            "item_probability": batch.augmentation_value,
            "next_item_probability": batch.next_augmentation_value,
            "action": action,
            "next_action": next_action,
            "position_reward": position_reward,
            "reward_mask": reward_mask,
            "time_diff": None,
            "not_terminal": ~batch.terminal,
        })


REPLAY_BUFFER_MAKER_MAP = {
    rlt.DiscreteDqnInput: DiscreteDqnInputMaker,
    rlt.PolicyNetworkInput: PolicyNetworkInputMaker,
    rlt.MemoryNetworkInput: MemoryNetworkInputMaker,
    rlt.SlateQInput: SlateQInputMaker,
}


def make_replay_buffer_trainer_preprocessor(trainer, device, env):
    """trainer_preprocessor.py:32-69: pick the maker from the annotation of
    train_step_gen's `training_batch` parameter."""
    sig = inspect.signature(trainer.train_step_gen)
    assert list(sig.parameters.keys())[0] == "training_batch"
    training_batch_type = sig.parameters["training_batch"].annotation
    assert training_batch_type != inspect.Parameter.empty
    maker = REPLAY_BUFFER_MAKER_MAP[training_batch_type].create_for_env(env)

    def trainer_preprocessor(batch):
        return maker(batch).to(device)

    return trainer_preprocessor
