"""BatchConstrainedDQN (reagent/models/bcq.py:11-35): the act-time model of batch-constrained
Q-learning.  Scores are the q-network's, with -1e10 added to every action the imitator (the
behaviour policy) considers unlikely:

    r = softmax(imitator(state)) / max(softmax(imitator(state)))
    q = q_network(state) + (-1e10) * (r < bcq_drop_threshold)

forward() is three launches: the q-network's fused forward, the imitator's fused forward and
rb200_bcq_filter in its model mode."""
import torch

from .. import _lib
from ..core import types as rlt
from .base import ModelBase, require_cuda
from .fully_connected_network import FullyConnectedNetwork


class BatchConstrainedDQN(ModelBase):
    def __init__(self, state_dim, q_network, imitator_network, bcq_drop_threshold) -> None:
        super().__init__()
        assert state_dim > 0, "state_dim must be > 0, got {}".format(state_dim)
        if not isinstance(imitator_network, FullyConnectedNetwork):
            raise NotImplementedError(
                "the BCQ imitator must be a reagent_b200.models.FullyConnectedNetwork (its "
                "forward runs on the fused MLP kernel); got " + type(imitator_network).__name__)
        self.state_dim = state_dim
        self.q_network = q_network
        self.imitator_network = imitator_network
        self.invalid_action_penalty = -1e10
        self.bcq_drop_threshold = bcq_drop_threshold

    def input_prototype(self):
        return self.q_network.input_prototype()

    def forward(self, state: rlt.FeatureData) -> torch.Tensor:
        x = state.float_features
        require_cuda(x, type(self).__name__ + ".forward")
        q = self.q_network(state).contiguous().float()
        logits = self.imitator_network(x)
        if q.dim() != 2 or logits.shape != q.shape:
            raise ValueError(f"q-values {tuple(q.shape)} and imitator outputs "
                             f"{tuple(logits.shape)} must both be (batch, num_actions)")
        B, A = q.shape
        out = torch.empty_like(q)
        rc = _lib.lib().rb200_bcq_filter(logits.data_ptr(), B, A, float(self.bcq_drop_threshold),
                                         None, None, q.data_ptr(), out.data_ptr(),
                                         _lib.cur_stream())
        _lib.check(rc, "rb200_bcq_filter")
        return out
