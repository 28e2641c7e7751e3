"""Agent-side helpers (mirrors of the trajectory post-processing in xt/agent/ppo and the MuZero agents of xt/agent/muzero)."""
from .ppo import PPO, AtariPpo  # noqa: F401
from .muzero import Muzero, MuzeroAtari, search_predict_fn  # noqa: F401
