"""ImpalaMlp on the CUDA engine (xt/model/impala/impala_mlp.py:30-93)."""
from ..registry import Registers
from . import archs
from .impala_keras import ImpalaKerasModel

# xt/model/impala/default_config.py
LR = 0.0003
ENTROPY_LOSS = 0.01
HIDDEN_SIZE = 128
NUM_LAYERS = 1


@Registers.model
class ImpalaMlp(ImpalaKerasModel):
    """Dense(HIDDEN_SIZE, relu) x NUM_LAYERS -> softmax policy (A) + value (1); Keras Adam(LR)."""
    config = globals()
    clipnorm = None
    decay = 0.0

    def build_arch(self):
        return archs.impala_mlp(self.state_dim, self.action_dim, HIDDEN_SIZE, NUM_LAYERS)
