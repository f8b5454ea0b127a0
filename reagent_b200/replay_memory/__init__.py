from .circular_replay_buffer import ReplayBuffer  # noqa: F401
from .prioritized_replay_buffer import PrioritizedReplayBuffer  # noqa: F401
from .sum_tree import SumTree  # noqa: F401
from .device_replay import PrioritizedUpdate, PriorityShard  # noqa: F401
