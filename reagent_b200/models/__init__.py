from .arena import ParamArena, ScalarArena, arena_of  # noqa: F401
from .actor import FullyConnectedActor, GaussianFullyConnectedActor  # noqa: F401
from .base import ModelBase  # noqa: F401
from .bcq import BatchConstrainedDQN  # noqa: F401
from .categorical_dqn import CategoricalDQN  # noqa: F401
from .cem_planner import CEMNoise, CEMPlan, CEMPlannerNetwork  # noqa: F401
from .critic import FullyConnectedCritic  # noqa: F401
from .dqn import FullyConnectedDQN  # noqa: F401
from .dueling_q_network import DuelingQNetwork  # noqa: F401
from .fully_connected_network import (  # noqa: F401
    FloatFeatureFullyConnected,
    FullyConnectedNetwork,
)
from .seq2reward_model import Seq2RewardNetwork  # noqa: F401
from .seq2slate import (  # noqa: F401
    Seq2SlateMode,
    Seq2SlateOutputArch,
    Seq2SlateTransformerNet,
)
from .world_model import MDNRNN, LstmArena, MemoryNetwork  # noqa: F401
