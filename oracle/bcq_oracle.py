"""TEST INFRASTRUCTURE ONLY -- CPU restatement of batch-constrained Q-learning (BCQ) on top of
the DQN oracle in oracle/td_oracle.py.  Never imported by the product path.

PINNED: tests/test_bcq_cpu.py checks every function here against golden vectors that
oracle/make_bcq_golden.py produced by running the UNMODIFIED reference DQNTrainer with an
imitator and BCQConfig, and BatchConstrainedDQN.

BCQ only narrows a mask, so each function here filters the batch's mask and hands the batch to
the td_oracle function it wraps.
"""
from typing import Dict, Optional

import torch

from oracle import td_oracle as O


def bcq_filter(imitator: O.Net, x: torch.Tensor, thr: float):
    """get_valid_actions_from_imitator (reagent/training/imitator_training.py:12-25) for a torch
    imitator: returns (keep as float 0/1, filter values r = softmax / its row max)."""
    with torch.no_grad():
        p = torch.softmax(O.mlp(imitator, x), dim=1)
        r = p / p.max(keepdim=True, dim=1)[0]
    return (r >= thr).float(), r


def filtered_next_mask(batch: Dict[str, torch.Tensor], imitator: O.Net, thr: float):
    """possible_next_actions_mask.float() * keep(next_state) -- dqn_trainer.py:206-216."""
    keep, _ = bcq_filter(imitator, batch["next_state"], thr)
    return batch["possible_next_actions_mask"].float() * keep


def dqn_td_loss(q: O.Net, qt: O.Net, batch, *, imitator: O.Net, bcq_threshold: float,
                maxq: bool = True, **kw):
    """td_oracle.dqn_td_loss with the max-Q mask narrowed by the imitator (the SARSA branch
    ignores BCQ, dqn_trainer.py:221-227).  aux["next_mask"] is the mask the max ran over."""
    if maxq:
        batch = dict(batch, possible_next_actions_mask=filtered_next_mask(batch, imitator,
                                                                          bcq_threshold))
    td, aux = O.dqn_td_loss(q, qt, batch, maxq=maxq, **kw)
    aux["next_mask"] = (batch["possible_next_actions_mask"] if maxq else batch["next_action"]).float()
    return td, aux


def dqn_update(q: O.Net, qt: O.Net, adam: O.AdamState, batch, *, gamma, tau, imitator: O.Net,
               bcq_threshold: float, maxq: bool = True, **kw):
    """td_oracle.dqn_update with the BCQ filter.  Returns (loss, grads, aux)."""
    mask = None
    if maxq:
        mask = filtered_next_mask(batch, imitator, bcq_threshold)
        batch = dict(batch, possible_next_actions_mask=mask)
    loss, grads, aux = O.dqn_update(q, qt, adam, batch, gamma=gamma, tau=tau, maxq=maxq, **kw)
    aux["next_mask"] = mask
    return loss, grads, aux


def _cpe_batch(batch, imitator: Optional[O.Net], bcq_threshold, maxq):
    """The reference's `mask = batch_mask.float(); mask *= keep` writes the batch tensor itself
    exactly when it already is float32; only then does _calculate_cpes see the filtered mask."""
    m = batch["possible_next_actions_mask"]
    if imitator is not None and maxq and m.dtype == torch.float32:
        return dict(batch, possible_next_actions_mask=filtered_next_mask(batch, imitator,
                                                                         bcq_threshold))
    return batch


def dqn_cpe_losses(q, reward_net, qcpe, qcpe_t, batch, *, imitator: Optional[O.Net] = None,
                   bcq_threshold: Optional[float] = None, maxq: bool = True, **kw):
    """td_oracle.dqn_cpe_losses as DQNTrainer with BCQ evaluates them (see _cpe_batch)."""
    return O.dqn_cpe_losses(q, reward_net, qcpe, qcpe_t,
                            _cpe_batch(batch, imitator, bcq_threshold, maxq), maxq=maxq, **kw)


def dqn_cpe_update(q, reward_net, adam_r, qcpe, qcpe_t, adam_c, batch, *, tau,
                   imitator: Optional[O.Net] = None, bcq_threshold: Optional[float] = None,
                   maxq: bool = True, **kw):
    """td_oracle.dqn_cpe_update as DQNTrainer with BCQ runs it (see _cpe_batch)."""
    return O.dqn_cpe_update(q, reward_net, adam_r, qcpe, qcpe_t, adam_c,
                            _cpe_batch(batch, imitator, bcq_threshold, maxq), tau=tau, maxq=maxq,
                            **kw)


def model_forward(q: O.Net, imitator: O.Net, x: torch.Tensor, thr: float):
    """BatchConstrainedDQN.forward (reagent/models/bcq.py:26-35):
    q(x) + (-1e10) * (r < thr)."""
    keep, _ = bcq_filter(imitator, x, thr)
    with torch.no_grad():
        return O.mlp(q, x) + (-1e10) * (1.0 - keep)
