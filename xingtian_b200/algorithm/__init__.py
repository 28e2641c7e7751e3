"""Algorithm plugins (mirror of xt/algorithm)."""
from .base import Algorithm  # noqa: F401
from .ppo import PPO  # noqa: F401
from .impala_opt import IMPALAOpt  # noqa: F401
from .impala import IMPALA  # noqa: F401
from .dqn import DQN  # noqa: F401
from .replay_buffer import ReplayBuffer, DeviceReplayBuffer  # noqa: F401
from .muzero import Muzero  # noqa: F401
