"""Net builders with the reference's build_* signatures (reagent/net_builder/**): config
dataclass -> arena-backed model.  Normalization data only sizes the input/output dims
(get_num_output_features); serving wrappers (build_serving_module) are out of scope."""
from dataclasses import dataclass, field
from typing import List

from ..core.parameters import NormalizationData, TransformerParameters
from ..models import (CategoricalDQN, DuelingQNetwork, FullyConnectedActor,
                      FullyConnectedCritic, FullyConnectedDQN, GaussianFullyConnectedActor)
from ..models.fully_connected_network import FloatFeatureFullyConnected
from ..models.seq2slate import Seq2SlateOutputArch
from ..preprocessing.normalization import get_num_output_features


def _dim(normalization_data: NormalizationData) -> int:
    return get_num_output_features(normalization_data.dense_normalization_parameters)


@dataclass
class FullyConnected:
    """reagent/net_builder/discrete_dqn/fully_connected.py:16-46"""
    sizes: List[int] = field(default_factory=lambda: [256, 128])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    dropout_ratio: float = 0.0
    use_batch_norm: bool = False

    def build_q_network(self, state_feature_config, state_normalization_data: NormalizationData,
                        output_dim: int):
        return FullyConnectedDQN(state_dim=_dim(state_normalization_data), action_dim=output_dim,
                                 sizes=self.sizes, activations=self.activations,
                                 dropout_ratio=self.dropout_ratio,
                                 use_batch_norm=self.use_batch_norm)


@dataclass
class Dueling:
    """reagent/net_builder/discrete_dqn/dueling.py:16-40 (the default of the DiscreteDQN manager)"""
    sizes: List[int] = field(default_factory=lambda: [256, 128])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])

    def __post_init__(self):
        assert len(self.sizes) == len(self.activations), (
            f"Must have the same numbers of sizes and activations; got: "
            f"{self.sizes}, {self.activations}")

    def build_q_network(self, state_feature_config, state_normalization_data: NormalizationData,
                        output_dim: int):
        return DuelingQNetwork.make_fully_connected(_dim(state_normalization_data), output_dim,
                                                    self.sizes, self.activations)


@dataclass
class Quantile:
    """reagent/net_builder/quantile_dqn/quantile.py:15-44"""
    sizes: List[int] = field(default_factory=lambda: [256, 128])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    dropout_ratio: float = 0.0

    def build_q_network(self, state_normalization_data: NormalizationData, output_dim: int,
                        num_atoms: int):
        return FullyConnectedDQN(state_dim=_dim(state_normalization_data), action_dim=output_dim,
                                 sizes=self.sizes, activations=self.activations,
                                 num_atoms=num_atoms, dropout_ratio=self.dropout_ratio)


@dataclass
class DuelingQuantile:
    """reagent/net_builder/quantile_dqn/dueling_quantile.py:16-40"""
    sizes: List[int] = field(default_factory=lambda: [256, 128])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])

    def __post_init__(self):
        assert len(self.sizes) == len(self.activations), (
            f"Must have the same numbers of sizes and activations; got: {self.sizes}, {self.activations}")

    def build_q_network(self, state_normalization_data: NormalizationData, output_dim: int,
                        num_atoms: int):
        return DuelingQNetwork.make_fully_connected(
            _dim(state_normalization_data), output_dim, layers=self.sizes,
            activations=self.activations, num_atoms=num_atoms)


@dataclass
class Categorical:
    """reagent/net_builder/categorical_dqn/categorical.py:15-49"""
    sizes: List[int] = field(default_factory=lambda: [256, 128])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])

    def __post_init__(self):
        assert len(self.sizes) == len(self.activations), (
            f"Must have the same numbers of sizes and activations; got: {self.sizes}, {self.activations}")

    def build_q_network(self, state_normalization_data: NormalizationData, output_dim: int,
                        num_atoms: int, qmin: float, qmax: float):
        dist = FullyConnectedDQN(state_dim=_dim(state_normalization_data), action_dim=output_dim,
                                 sizes=self.sizes, activations=self.activations,
                                 num_atoms=num_atoms)
        return CategoricalDQN(dist, qmin=qmin, qmax=qmax, num_atoms=num_atoms)


@dataclass
class ParametricFullyConnected:
    """reagent/net_builder/parametric_dqn/fully_connected.py:16-54 (the SAC / TD3 critics)"""
    sizes: List[int] = field(default_factory=lambda: [128, 64])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    use_batch_norm: bool = False
    use_layer_norm: bool = False
    final_activation: str = "linear"

    def build_q_network(self, state_normalization_data: NormalizationData,
                        action_normalization_data: NormalizationData, output_dim: int = 1):
        return FullyConnectedCritic(
            _dim(state_normalization_data), _dim(action_normalization_data), sizes=self.sizes,
            activations=self.activations, use_batch_norm=self.use_batch_norm,
            use_layer_norm=self.use_layer_norm, output_dim=output_dim,
            final_activation=self.final_activation)


@dataclass
class GaussianFullyConnected:
    """reagent/net_builder/continuous_actor/gaussian_fully_connected.py:23-82"""
    sizes: List[int] = field(default_factory=lambda: [128, 64])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    use_batch_norm: bool = False
    use_layer_norm: bool = False
    use_l2_normalization: bool = False

    def build_actor(self, state_feature_config, state_normalization_data: NormalizationData,
                    action_normalization_data: NormalizationData):
        return GaussianFullyConnectedActor(
            state_dim=_dim(state_normalization_data), action_dim=_dim(action_normalization_data),
            sizes=self.sizes, activations=self.activations, use_batch_norm=self.use_batch_norm,
            use_layer_norm=self.use_layer_norm, use_l2_normalization=self.use_l2_normalization)


@dataclass
class ActorFullyConnected:
    """reagent/net_builder/continuous_actor/fully_connected.py:22-76"""
    sizes: List[int] = field(default_factory=lambda: [128, 64])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    use_batch_norm: bool = False
    action_activation: str = "tanh"
    exploration_variance: float = None

    def build_actor(self, state_feature_config, state_normalization_data: NormalizationData,
                    action_normalization_data: NormalizationData):
        return FullyConnectedActor(
            state_dim=_dim(state_normalization_data), action_dim=_dim(action_normalization_data),
            sizes=self.sizes, activations=self.activations, use_batch_norm=self.use_batch_norm,
            action_activation=self.action_activation,
            exploration_variance=self.exploration_variance)


@dataclass
class DiscreteActorFullyConnected:
    """reagent/net_builder/discrete_actor/fully_connected.py:22-71: one logit per action (the
    actor of DiscreteCRRTrainer)."""
    sizes: List[int] = field(default_factory=lambda: [128, 64])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    use_batch_norm: bool = False
    use_layer_norm: bool = False
    action_activation: str = "tanh"
    exploration_variance: float = None

    def __post_init__(self):
        assert len(self.sizes) == len(self.activations), (
            f"Must have the same numbers of sizes and activations; got: "
            f"{self.sizes}, {self.activations}")
        if self.use_layer_norm:
            raise NotImplementedError("layer norm is out of scope of reagent_b200 (SURVEY.md M1)")

    def build_actor(self, state_normalization_data: NormalizationData, num_actions: int):
        return FullyConnectedActor(
            state_dim=_dim(state_normalization_data), action_dim=num_actions, sizes=self.sizes,
            activations=self.activations, use_batch_norm=self.use_batch_norm,
            action_activation=self.action_activation,
            exploration_variance=self.exploration_variance)


@dataclass
class ValueFullyConnected:
    """reagent/net_builder/value/fully_connected.py:16-44 (the SAC state-value network)"""
    sizes: List[int] = field(default_factory=lambda: [256, 128])
    activations: List[str] = field(default_factory=lambda: ["relu", "relu"])
    use_layer_norm: bool = False

    def __post_init__(self):
        assert len(self.sizes) == len(self.activations), (
            f"Must have the same numbers of sizes and activations; got: {self.sizes}, {self.activations}")

    def build_value_network(self, state_normalization_data: NormalizationData,
                            output_dim: int = 1):
        return FloatFeatureFullyConnected(
            state_dim=_dim(state_normalization_data), output_dim=output_dim, sizes=self.sizes,
            activations=self.activations, use_layer_norm=self.use_layer_norm)


@dataclass
class Seq2RewardNetBuilder:
    """reagent/net_builder/value/seq2reward_rnn.py"""
    action_dim: int = 2
    num_hiddens: int = 64
    num_hidden_layers: int = 2

    def build_value_network(self, state_normalization_data: NormalizationData):
        from ..models.seq2reward_model import Seq2RewardNetwork

        return Seq2RewardNetwork(state_dim=_dim(state_normalization_data),
                                 action_dim=self.action_dim, num_hiddens=self.num_hiddens,
                                 num_hidden_layers=self.num_hidden_layers)


@dataclass
class SlateRankingTransformer:
    """reagent/net_builder/slate_ranking/slate_ranking_transformer.py"""
    output_arch: Seq2SlateOutputArch = Seq2SlateOutputArch.AUTOREGRESSIVE
    temperature: float = 1.0
    transformer: TransformerParameters = field(
        default_factory=lambda: TransformerParameters(num_heads=2, dim_model=16,
                                                      dim_feedforward=16, num_stacked_layers=2))

    def build_slate_ranking_network(self, state_dim, candidate_dim, candidate_size, slate_size):
        from ..models.seq2slate import Seq2SlateTransformerNet

        return Seq2SlateTransformerNet(
            state_dim=state_dim, candidate_dim=candidate_dim,
            num_stacked_layers=self.transformer.num_stacked_layers,
            num_heads=self.transformer.num_heads, dim_model=self.transformer.dim_model,
            dim_feedforward=self.transformer.dim_feedforward, max_src_seq_len=candidate_size,
            max_tgt_seq_len=slate_size, output_arch=self.output_arch,
            temperature=self.temperature, state_embed_dim=self.transformer.state_embed_dim)
