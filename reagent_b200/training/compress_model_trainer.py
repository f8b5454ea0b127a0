"""CompressModelTrainer (reagent/training/world_model/compress_model_trainer.py): fits an MLP
policy to the Seq2Reward plan.  Per update:

  rb200_mlp_forward               compress_model_network(state[0])
  rb200_seq2reward_plan           get_Q over the prefix tree: the regression target
  rb200_seq2reward_compress_head  MSE, dL/dout and the argmax accuracy
  rb200_mlp_backward, rb200_mlp_wgrad

then FusedAdam at compress_model_learning_rate.
"""
import logging

import torch

from .. import _lib
from ..core import types as rlt
from ..core.parameters import Seq2RewardTrainerParameters
from ..core.types import FeatureData
from ..models.fully_connected_network import FloatFeatureFullyConnected
from ..models.seq2reward_model import Seq2RewardNetwork
from ..optimizer import FusedAdam
from .reagent_lightning_module import ReAgentLightningModule
from .seq2reward_trainer import _check_permutations, gen_permutations
from .workspace import NetWorkspace, backward_wgrad, param_grads

logger = logging.getLogger(__name__)


class CompressModelTrainer(ReAgentLightningModule):
    """Trainer for fitting Seq2Reward planning outcomes to a neural network-based policy"""

    def __init__(self, compress_model_network: FloatFeatureFullyConnected,
                 seq2reward_network: Seq2RewardNetwork, params: Seq2RewardTrainerParameters):
        super().__init__()
        if not isinstance(compress_model_network, FloatFeatureFullyConnected) or \
                compress_model_network.num_atoms is not None:
            raise NotImplementedError("CompressModelTrainer needs a reagent_b200.models."
                                      "FloatFeatureFullyConnected without atoms; got "
                                      + type(compress_model_network).__name__)
        if not isinstance(seq2reward_network, Seq2RewardNetwork):
            raise NotImplementedError("CompressModelTrainer needs a reagent_b200.models."
                                      "Seq2RewardNetwork; got " + type(seq2reward_network).__name__)
        self.compress_model_network = compress_model_network
        self.seq2reward_network = seq2reward_network
        self.params = params
        # permutations used to do planning
        self.all_permut = gen_permutations(params.multi_steps, len(self.params.action_names))
        self._ws = None

    def configure_optimizers(self):
        """[Adam(compress_model_network, compress_model_learning_rate)]"""
        return [FusedAdam(self.compress_model_network.parameters(),
                          lr=self.params.compress_model_learning_rate)]

    @staticmethod
    def extract_state_first_step(batch):
        return FeatureData(batch.state.float_features[0])

    def _step(self, batch: rlt.MemoryNetworkInput, train: bool):
        """Device vector [mse, accuracy] (and with `train` the gradient partials); no host
        synchronisation."""
        state = batch.state.float_features
        if state.dim() != 3 or not state.is_cuda:
            raise ValueError(f"CompressModelTrainer: state must be a [T, B, state_dim] CUDA "
                             f"tensor, got {tuple(state.shape)} on {state.device}")
        _lib.require_current_device(state.device)
        state0 = state[0].float().contiguous()
        B = state0.shape[0]
        ar = self.compress_model_network.arena
        A = ar.dims[-1]
        k, pa = _check_permutations(self.all_permut)
        if pa != A:
            raise ValueError(f"CompressModelTrainer: {pa} actions in the plan, {A} outputs")
        ws = self._ws
        if ws is None or ws["B"] != B or ws["dev"] != state.device:
            ws = self._ws = {
                "B": B, "dev": state.device, "net": NetWorkspace(ar, B, state.device),
                "out": torch.empty(B, A, device=state.device),
                "loss_partials": torch.zeros(2 * -(-B // 256), device=state.device),
                "counter": torch.zeros(1, dtype=torch.int32, device=state.device),
                "loss": torch.zeros(2, device=state.device)}
        ar.forward(state0, ws["out"], save=ws["net"] if train else None)
        q = self.seq2reward_network.plan(state0, k)[0]
        a = _lib.Seq2rewardCompressArgsT()
        a.batch, a.num_action = B, A
        a.out, a.q = ws["out"].data_ptr(), q.data_ptr()
        a.dout = ws["net"].dz[-1].data_ptr() if train else None
        a.loss_partials, a.tile_counter = ws["loss_partials"].data_ptr(), ws["counter"].data_ptr()
        a.out_loss = ws["loss"].data_ptr()
        _lib.check(_lib.lib().rb200_seq2reward_compress_head(a, _lib.cur_stream()),
                   "rb200_seq2reward_compress_head")
        if train:
            backward_wgrad(ar, ws["net"], state0, B)
        ws["q"] = q
        return ws["loss"]

    def get_loss(self, batch: rlt.MemoryNetworkInput):
        """(mse, accuracy) as device scalars."""
        loss = self._step(batch, train=False).clone()
        return loss[0], loss[1]

    def train_step_gen(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int):
        loss = self._step(training_batch, train=True)
        if self.has_real_reporter:
            detached_loss, accuracy = loss.cpu().tolist()
            logger.info(f"Seq2Reward Compress trainer MSE/Accuracy: {detached_loss}, {accuracy}")
            self.reporter.log(mse_loss=detached_loss, accuracy=accuracy)
        yield self.fused_loss(loss[0])

    def train_batch(self, training_batch: rlt.MemoryNetworkInput, batch_idx: int = 0):
        """Fast path: the update of train_step_gen plus one FusedAdam launch, with no host
        synchronisation.  Returns the device vector [mse, accuracy]."""
        loss = self._step(training_batch, train=True)
        self.adam_step(self.compress_model_network.arena)
        self.all_batches_processed += 1
        return loss

    @torch.no_grad()
    def validation_step(self, batch: rlt.MemoryNetworkInput, batch_idx: int):
        mse, acc = self.get_loss(batch)
        detached_loss = mse.item()
        acc = acc.item()
        # shape: batch_size, action_dim
        q_values_all_action_all_data = self._ws["out"].cpu()
        q_values = q_values_all_action_all_data.mean(0).tolist()
        action_distribution = torch.bincount(torch.argmax(q_values_all_action_all_data, dim=1),
                                             minlength=len(self.params.action_names))
        action_distribution = (action_distribution.float()
                               / torch.sum(action_distribution)).tolist()
        if self.has_real_reporter:
            self.reporter.log(eval_mse_loss=detached_loss, eval_accuracy=acc,
                              eval_q_values=[q_values],
                              eval_action_distribution=[action_distribution])
        return (detached_loss, q_values, action_distribution, acc)

    def warm_start_components(self):
        return []

    def compress_grads(self):
        """Per-parameter gradients of the last fused backward (inspection / tests)."""
        net = self.compress_model_network
        return param_grads(net.arena, list(net.parameters()))
