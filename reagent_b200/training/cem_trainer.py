"""CEMTrainer (reagent/training/cem_trainer.py): an ensemble of world models, each trained by
its own MDNRNNTrainer, and the cross-entropy-method planner that plans with them.

The idea is inspired by: https://arxiv.org/abs/1805.12114
"""
from typing import List

import torch.nn as nn

from ..core import types as rlt
from ..core.parameters import CEMTrainerParameters
from ..models.cem_planner import CEMPlannerNetwork
from .mdnrnn_trainer import MDNRNNTrainer
from .reagent_lightning_module import ReAgentLightningModule


class CEMTrainer(ReAgentLightningModule):
    def __init__(self, cem_planner_network: CEMPlannerNetwork,
                 world_model_trainers: List[MDNRNNTrainer],
                 parameters: CEMTrainerParameters) -> None:
        super().__init__()
        self.cem_planner_network = cem_planner_network
        self.world_model_trainers = nn.ModuleList(world_model_trainers)

    def configure_optimizers(self):
        """Every world-model trainer's optimizers, in order.  They are the trainers' own (their
        optimizers()), so the generator loop and train_batch step the same Adam state."""
        return [o for t in self.world_model_trainers for o in t.optimizers()]

    def train_step_gen(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int):
        for t in self.world_model_trainers:
            yield from t.train_step_gen(training_batch, batch_idx)

    def train_batch(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int = 0):
        """Fast path: each world-model trainer's train_batch on the batch, in order, with no
        host synchronisation.  Returns their device loss vectors [gmm, bce, mse, loss] (each
        overwritten by that trainer's next step)."""
        losses = [t.train_batch(training_batch, batch_idx) for t in self.world_model_trainers]
        self.all_batches_processed += 1
        return losses
