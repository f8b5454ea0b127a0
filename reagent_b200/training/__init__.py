from .behavioral_cloning_trainer import BehavioralCloningTrainer  # noqa: F401
from .c51_trainer import C51Trainer  # noqa: F401
from .cem_trainer import CEMTrainer  # noqa: F401
from .compress_model_trainer import CompressModelTrainer  # noqa: F401
from .discrete_crr_trainer import DiscreteCRRTrainer  # noqa: F401
from .dqn_trainer import BCQConfig, DQNTrainer  # noqa: F401
from .loop import run_update  # noqa: F401
from .mdnrnn_trainer import MDNRNNTrainer  # noqa: F401
from .parametric_dqn_trainer import ParametricDQNTrainer  # noqa: F401
from .ppo_trainer import PPOTrainer  # noqa: F401
from .qrdqn_trainer import QRDQNTrainer  # noqa: F401
from .reagent_lightning_module import ReAgentLightningModule  # noqa: F401
from .reinforce_trainer import ReinforceTrainer  # noqa: F401
from .sac_trainer import CRRWeightFn, SACTrainer  # noqa: F401
from .seq2reward_trainer import (  # noqa: F401
    Seq2RewardTrainer,
    gen_permutations,
    get_Q,
    get_step_prediction,
    plan_short_sequence_q,
)
from .slate_q_trainer import NextSlateValueNormMethod, SlateQTrainer  # noqa: F401
from .td3_trainer import TD3Trainer  # noqa: F401
