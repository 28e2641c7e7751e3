"""xingtian_b200 -- H100 (sm_90a) engine for XingTian's actor-learner hot path.

Importing this package registers drop-in replacements for the reference's hot-path plugins
(``PpoCnn``, ``PpoMlp``, ``ImpalaCnnOpt``, ``ImpalaMlp``, ``ImpalaCnn``, ``DqnCnn``, ``DqnMlp``, ``MuzeroCnn``, ``MuzeroMlp`` models; ``PPO``,
``IMPALAOpt``, ``IMPALA``, ``DQN``, ``Muzero`` algorithms; ``PPO``/``AtariPpo``/``Muzero``/``MuzeroAtari`` agents; ``ShareByPlasma``/``CommByZmq`` comm backends) under the same registry keys.  All numerics run
in libxtb200.so (hand-written CUDA); there is no CPU fallback."""
from .registry import Registers, import_config, model_builder, alg_builder, install  # noqa: F401
from . import model, algorithm, agent, ipc  # noqa: F401  (registration side effects)

__all__ = ["Registers", "import_config", "model_builder", "alg_builder", "install"]
