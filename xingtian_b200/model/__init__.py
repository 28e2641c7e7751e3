"""Model plugins (mirror of xt/model)."""
from .base import XTModel  # noqa: F401
from .ppo import PPO, PpoCnn, PpoMlp  # noqa: F401
from .impala import ImpalaCnnOpt  # noqa: F401
from .dqn import DqnCnn, DqnMlp  # noqa: F401
from .impala_mlp import ImpalaMlp  # noqa: F401
from .impala_cnn import ImpalaCnn  # noqa: F401
from .muzero import MuzeroCnn, MuzeroMlp, MuzeroModel  # noqa: F401
