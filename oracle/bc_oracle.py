"""TEST INFRASTRUCTURE ONLY -- CPU restatement of BehavioralCloningTrainer
(reagent/training/behavioral_cloning_trainer.py:17-83) on the networks of oracle/td_oracle.py.
Never imported by the product path.

PINNED: tests/test_bc_cpu.py checks it against golden vectors that oracle/make_bc_golden.py
produced by running the UNMODIFIED reference trainer.

Labels are each row's own action, `action.argmax(dim=1)`; on the golden inputs (B == A,
involutive label permutations) that equals the reference's `action.max(dim=0)[1]`.
"""
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import td_oracle as O

INVALID_ACTION_CONSTANT = -1e10


def masked_logits(net: O.Net, state: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """FullyConnectedDQN.forward(state, possible_actions_mask) -- reagent/models/dqn.py:55-63."""
    return O.mlp(net, state) + INVALID_ACTION_CONSTANT * (1 - mask.float())


def bc_loss(net: O.Net, batch: Dict[str, torch.Tensor]):
    """CrossEntropyLoss(reduction="mean")(masked logits, labels) -- :38-56.
    Returns (loss, logits)."""
    logits = masked_logits(net, batch["state"], batch["possible_actions_mask"])
    return F.cross_entropy(logits, batch["action"].argmax(dim=1)), logits


def bc_update(net: O.Net, adam: O.AdamState, batch):
    """One update (loss, backward, Adam).  Returns (loss, grads, logits)."""
    params = O.net_params(net)
    loss, logits = bc_loss(net, batch)
    grads = torch.autograd.grad(loss, params)
    adam.step(params, grads)
    return float(loss.detach()), [g.detach() for g in grads], logits.detach()
