"""Hyper-parameter dataclasses of the hot path, same field names and defaults as the
reference (reagent/core/parameters.py:46-67, :118-120, :138-152).  The reference's
pydantic/registry config machinery is out of scope (SURVEY.md section 2 row 6); plain frozen
dataclasses carry the same values."""
import enum
from dataclasses import dataclass, field
from typing import Dict, List, Optional

CONTINUOUS_TRAINING_ACTION_RANGE = (-1.0, 1.0)  # reagent/core/parameters.py:20


@dataclass(frozen=True)
class RLParameters:
    gamma: float = 0.9
    epsilon: float = 0.1
    target_update_rate: float = 0.001
    maxq_learning: bool = True
    reward_boost: Optional[Dict[str, float]] = None
    temperature: float = 0.01
    softmax_policy: bool = False
    use_seq_num_diff_as_time_diff: bool = False
    q_network_loss: str = "mse"
    set_missing_value_to_zero: bool = False
    tensorboard_logging_freq: int = 0
    predictor_atol_check: float = 0.0
    predictor_rtol_check: float = 5e-5
    time_diff_unit_length: float = 1.0
    multi_steps: Optional[int] = None
    ratio_different_predictions_tolerance: float = 0

    def asdict(self):
        import dataclasses

        return dataclasses.asdict(self)


@dataclass(frozen=True)
class EvaluationParameters:
    calc_cpe_in_training: bool = True


@dataclass(frozen=True)
class NormalizationParameters:
    feature_type: str
    boxcox_lambda: Optional[float] = None
    boxcox_shift: Optional[float] = None
    mean: Optional[float] = None
    stddev: Optional[float] = None
    possible_values: Optional[List[int]] = None
    quantiles: Optional[List[float]] = None
    min_value: Optional[float] = None
    max_value: Optional[float] = None


@dataclass
class NormalizationData:
    dense_normalization_parameters: Dict[int, NormalizationParameters] = field(default_factory=dict)


@dataclass(frozen=True)
class MDNRNNTrainerParameters:
    hidden_size: int = 64
    num_hidden_layers: int = 2
    learning_rate: float = 0.001
    num_gaussians: int = 5
    # weight in calculating world-model loss
    reward_loss_weight: float = 1.0
    next_state_loss_weight: float = 1.0
    not_terminal_loss_weight: float = 1.0
    fit_only_one_next_step: bool = False
    action_dim: int = 2
    action_names: Optional[List[str]] = None
    multi_steps: int = 1


@dataclass(frozen=True)
class Seq2RewardTrainerParameters:
    learning_rate: float = 0.001
    multi_steps: int = 1
    action_names: List[str] = field(default_factory=lambda: [])
    compress_model_learning_rate: float = 0.001
    gamma: float = 1.0
    view_q_value: bool = False
    step_predict_net_size: int = 64
    reward_boost: Optional[Dict[str, float]] = None


@dataclass(frozen=True)
class CEMTrainerParameters:
    plan_horizon_length: int = 0
    num_world_models: int = 0
    cem_population_size: int = 0
    cem_num_iterations: int = 0
    ensemble_population_size: int = 0
    num_elites: int = 0
    mdnrnn: MDNRNNTrainerParameters = field(default_factory=MDNRNNTrainerParameters)
    rl: RLParameters = field(default_factory=RLParameters)
    alpha: float = 0.25
    epsilon: float = 0.001


class SlateOptMethod(enum.Enum):
    """reagent/core/parameters.py:33-36"""
    GREEDY = "greedy"
    TOP_K = "top_k"
    EXACT = "exact"


@dataclass(frozen=True)
class SlateOptParameters:
    method: SlateOptMethod = SlateOptMethod.TOP_K


def _default_optimizer():
    from ..optimizer import Optimizer__Union

    return Optimizer__Union.default()


def _norm_by_current_slate_size():
    from ..training.slate_q_trainer import NextSlateValueNormMethod

    return NextSlateValueNormMethod.NORM_BY_CURRENT_SLATE_SIZE


@dataclass(frozen=True)
class SlateQTrainerParameters:
    """The arguments of SlateQTrainer after the networks and slate_size, with the reference's
    defaults (the reference generates this class from the trainer's __init__).  The optimizer
    is an Optimizer__Union and the norm method a NextSlateValueNormMethod
    (reagent_b200.training.slate_q_trainer); both defaults are made on first use, since those
    modules import this one."""
    rl: RLParameters = field(default_factory=lambda: RLParameters(maxq_learning=False))
    optimizer: object = field(default_factory=_default_optimizer)
    slate_opt_parameters: Optional[SlateOptParameters] = None
    discount_time_scale: Optional[float] = None
    single_selection: bool = True
    next_slate_value_norm_method: object = field(default_factory=_norm_by_current_slate_size)
    minibatch_size: int = 1024
    evaluation: EvaluationParameters = field(
        default_factory=lambda: EvaluationParameters(calc_cpe_in_training=False))

    def asdict(self):
        import dataclasses

        return {f.name: getattr(self, f.name) for f in dataclasses.fields(self)}


@dataclass(frozen=True)
class TransformerParameters:
    """reagent/core/parameters.py:183: the shape of a Seq2Slate transformer."""
    num_heads: int = 1
    dim_model: int = 64
    dim_feedforward: int = 32
    num_stacked_layers: int = 2
    state_embed_dim: Optional[int] = None


class NormalizationKey:
    STATE = "state"
    ACTION = "action"
    ITEM = "item"
