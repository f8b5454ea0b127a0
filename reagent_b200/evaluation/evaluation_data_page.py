"""EvaluationDataPage (reagent/evaluation/evaluation_data_page.py) for discrete-action DQN and
CRR trainers.  The page lives on the device its batches came from: the networks run on the fused
MLP kernels, rb200_ope_page derives the per-row fields, and sort / compute_values / validate run
on the device (the sort is torch's stable sort; the episode recursions and checks are kernels)."""
from dataclasses import dataclass, fields, replace
from typing import Optional

import numpy as np
import torch

from ..core import types as rlt
from . import _ope


@dataclass
class EvaluationDataPage:
    mdp_id: Optional[torch.Tensor]
    sequence_number: Optional[torch.Tensor]
    logged_propensities: torch.Tensor
    logged_rewards: torch.Tensor
    action_mask: torch.Tensor
    model_propensities: torch.Tensor
    model_rewards: torch.Tensor
    model_rewards_for_logged_action: torch.Tensor
    model_values: Optional[torch.Tensor] = None
    possible_actions_mask: Optional[torch.Tensor] = None
    optimal_q_values: Optional[torch.Tensor] = None
    eval_action_idxs: Optional[torch.Tensor] = None
    logged_values: Optional[torch.Tensor] = None
    logged_metrics: Optional[torch.Tensor] = None
    logged_metrics_values: Optional[torch.Tensor] = None
    model_metrics: Optional[torch.Tensor] = None
    model_metrics_for_logged_action: Optional[torch.Tensor] = None
    model_metrics_values: Optional[torch.Tensor] = None
    model_metrics_values_for_logged_action: Optional[torch.Tensor] = None
    possible_actions_state_concat: Optional[torch.Tensor] = None
    contexts: Optional[torch.Tensor] = None

    def _replace(self, **kwargs):
        page = replace(self, **kwargs)
        if "mdp_id" not in kwargs and "sequence_number" not in kwargs and "_episodes" in self.__dict__:
            page.__dict__["_episodes"] = self.__dict__["_episodes"]
        return page

    def cpu(self):
        return self._map(lambda t: t.cpu())

    def _map(self, fn):
        return EvaluationDataPage(**{
            f.name: (fn(getattr(self, f.name)) if isinstance(getattr(self, f.name), torch.Tensor)
                     else getattr(self, f.name)) for f in fields(EvaluationDataPage)})

    @classmethod
    def create_from_training_batch(cls, tdb, trainer, reward_network=None):
        if isinstance(tdb, rlt.DiscreteDqnInput):
            extras = tdb.extras
            return cls.create_from_tensors_dqn(
                trainer, extras.mdp_id, extras.sequence_number, tdb.state, tdb.action,
                extras.action_probability, tdb.reward, tdb.possible_actions_mask,
                metrics=extras.metrics)
        raise NotImplementedError(f"training_input type: {type(tdb)}")

    @classmethod
    @torch.no_grad()
    def create_from_tensors_dqn(cls, trainer, mdp_ids, sequence_numbers, states, actions,
                                propensities, rewards, possible_actions_mask, metrics=None):
        """evaluation_data_page.py:309-462.  model_outputs come from
        trainer.page_model_outputs (q_network for DQN, the actor for CRR); the reward
        network and q_network_cpe run on the fused MLP forward; rb200_ope_page computes the
        boosted rewards, the propensities, eval_action_idxs and the logged-action gathers."""
        if trainer.reward_network is None or trainer.q_network_cpe is None:
            raise ValueError("CPE needs calc_cpe_in_training=True: the page is built from the "
                             "reward network and q_network_cpe")
        x = states.float_features if isinstance(states, rlt.FeatureData) else states
        dev = trainer.reward_network.arena.flat.device
        x = _ope.f32(x, "state")
        if x.device != dev:
            raise ValueError(f"the batch is on {x.device}, the trainer's networks on {dev}")
        n, A = x.shape[0], trainer.num_actions
        if not 0 < n <= _ope.MAX_ROWS:
            raise ValueError(f"an evaluation page holds 1 to {_ope.MAX_ROWS} rows, got {n}")
        MA = len(trainer.metrics_to_score) * A
        K = MA // A - 1
        model_outputs = trainer.page_model_outputs(rlt.FeatureData(x))
        model_outputs = _ope.f32(model_outputs, "model outputs")
        if model_outputs.shape != (n, A):
            raise ValueError(f"model outputs have shape {tuple(model_outputs.shape)}, want {(n, A)}")
        reward_out = torch.empty(n, MA, device=dev)
        qcpe_out = torch.empty(n, MA, device=dev)
        for net, out in ((trainer.reward_network, reward_out), (trainer.q_network_cpe, qcpe_out)):
            net.arena.refresh()
            net.arena.forward(x, out)
        action_mask = _ope.f32(actions, "action")
        pam = _ope.f32(possible_actions_mask, "possible_actions_mask")
        if action_mask.shape != (n, A) or pam.shape != (n, A):
            raise ValueError(f"action and possible_actions_mask must have shape {(n, A)}")
        reward = _ope.f32(rewards, "reward").reshape(-1)
        boost = trainer.reward_boosts.reshape(-1).float().contiguous()
        boosted = torch.empty(n, 1, device=dev)
        prop = torch.empty(n, A, device=dev)
        eval_idx = torch.empty(n, 1, dtype=torch.int64, device=dev)
        mr_logged = torch.empty(n, 1, device=dev)
        mm_logged = torch.empty(n, K, device=dev) if K else None
        mmv_logged = torch.empty(n, K, device=dev) if K else None
        _ope._call("rb200_ope_page", n, A, K, model_outputs.data_ptr(), reward_out.data_ptr(),
                   qcpe_out.data_ptr(), pam.data_ptr(), action_mask.data_ptr(), reward.data_ptr(),
                   boost.data_ptr(), float(trainer.rl_temperature),
                   boosted.data_ptr(), prop.data_ptr(), eval_idx.data_ptr(), mr_logged.data_ptr(),
                   None if mm_logged is None else mm_logged.data_ptr(),
                   None if mmv_logged is None else mmv_logged.data_ptr())
        return cls(
            mdp_id=mdp_ids,
            sequence_number=sequence_numbers,
            logged_propensities=propensities,
            logged_rewards=boosted,
            action_mask=action_mask,
            model_rewards=reward_out[:, :A],
            model_rewards_for_logged_action=mr_logged,
            model_values=qcpe_out[:, :A],
            model_metrics_values=qcpe_out[:, A:] if K else None,
            model_metrics_values_for_logged_action=mmv_logged,
            model_propensities=prop,
            logged_metrics=metrics,
            model_metrics=reward_out[:, A:],
            model_metrics_for_logged_action=mm_logged,
            logged_values=None,
            logged_metrics_values=None,
            possible_actions_mask=possible_actions_mask,
            optimal_q_values=model_outputs,
            eval_action_idxs=eval_idx,
        )

    def append(self, edp):
        """Rows of `edp` after this page's, field by field (torch.cat on the fields' device).
        A field must be present in both pages or in neither."""
        merged = {}
        for f in fields(EvaluationDataPage):
            a, b = getattr(self, f.name), getattr(edp, f.name)
            if (a is None) != (b is None):
                raise AssertionError(f"cannot append pages that disagree on field {f.name}")
            if a is None:
                merged[f.name] = None
            elif isinstance(a, np.ndarray):
                merged[f.name] = np.concatenate([a, b])
            elif isinstance(a, torch.Tensor):
                merged[f.name] = torch.cat([a, b])
            else:
                raise TypeError(f"field {f.name} holds a {type(a).__name__}")
        return EvaluationDataPage(**merged)

    def sort(self):
        """Rows ordered by (mdp_id, sequence_number, original row): two stable sorts."""
        _ope.check_ids(self.mdp_id, self.sequence_number)
        order = torch.argsort(self.sequence_number.reshape(-1), stable=True)
        order = order[torch.argsort(self.mdp_id.reshape(-1)[order], stable=True)]
        return self._map(lambda t: t[order])

    def compute_values(self, gamma: float):
        assert self.mdp_id is not None and self.sequence_number is not None
        ep = _ope.episodes(self)
        logged_values = self._values(ep, self.logged_rewards, gamma)
        logged_metrics_values = (None if self.logged_metrics is None
                                 else self._values(ep, self.logged_metrics, gamma))
        return self._replace(logged_values=logged_values,
                             logged_metrics_values=logged_metrics_values)

    @staticmethod
    def _values(ep, x, gamma):
        x = _ope.f32(x, "rewards")
        out = torch.empty_like(x)
        disc = ep.step_discounts(gamma)
        _ope._call("rb200_ope_logged_values", ep.num, ep.off.data_ptr(), disc.data_ptr(),
                   x.shape[1], x.data_ptr(), out.data_ptr())
        return out

    @staticmethod
    def compute_values_for_mdps(rewards, mdp_ids, sequence_numbers, gamma):
        """values[r, 0] += values[r+1, 0] * gamma ** (seq[r+1] - seq[r]) backwards inside each
        run of equal mdp_id, in float32.  Only column 0 recurses, as in the reference (its
        metrics' other columns are returned unchanged)."""
        return EvaluationDataPage._values(_ope.Episodes(mdp_ids, sequence_numbers), rewards, gamma)

    def validate(self):
        """Shape checks of every field the estimators read, then the episode checks: inside each
        run of equal mdp_id the sequence numbers increase, and no mdp_id forms two runs."""
        n, A = self.model_propensities.shape
        expect = {"logged_propensities": 1, "logged_rewards": 1, "logged_values": 1,
                  "model_propensities": A, "model_rewards": A, "model_values": A,
                  "action_mask": A}
        if self.logged_metrics is not None:
            m = self.logged_metrics.shape[1]
            expect.update(logged_metrics=m, logged_metrics_values=m, model_metrics=m * A,
                          model_metrics_values=m * A)
        for name, cols in expect.items():
            shape = tuple(getattr(self, name).shape)
            assert shape == (n, cols), f"{name} has shape {shape}, expected {(n, cols)}"
        ep = _ope.episodes(self)
        if ep.first_bad_row >= 0:
            i = ep.first_bad_row
            seq = self.sequence_number.reshape(-1)
            raise AssertionError(
                f"For mdp_id {int(self.mdp_id.reshape(-1)[i])}, got {int(seq[i])} <= "
                f"{int(seq[i - 1])}.Sequence number must be in increasing order.")
        unique = int(torch.unique(self.mdp_id.reshape(-1)).numel())
        assert unique == ep.runs, "MDPs are broken up. {} vs {}".format(unique, ep.runs)

    def set_metric_as_reward(self, i: int, num_actions: int):
        """A page that scores metric `i` as the reward: its logged column, logged values and
        the i-th `num_actions` block of the model's metric rewards and values; the metric fields
        themselves are dropped."""
        for name in ("logged_metrics", "logged_metrics_values", "model_metrics",
                     "model_metrics_values"):
            assert getattr(self, name) is not None, f"{name} is needed to score a metric"
        block = slice(i * num_actions, (i + 1) * num_actions)
        return self._replace(logged_rewards=self.logged_metrics[:, i:i + 1],
                             logged_values=self.logged_metrics_values[:, i:i + 1],
                             model_rewards=self.model_metrics[:, block],
                             model_values=self.model_metrics_values[:, block],
                             logged_metrics=None, logged_metrics_values=None,
                             model_metrics=None, model_metrics_values=None)
