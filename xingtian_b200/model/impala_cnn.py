"""ImpalaCnn on the CUDA engine (xt/model/impala/impala_cnn.py:32-108)."""
from ..registry import Registers
from . import archs
from .impala_keras import ImpalaKerasModel

# xt/model/impala/default_config.py
LR = 0.0003
ENTROPY_LOSS = 0.01


@Registers.model
class ImpalaCnn(ImpalaKerasModel):
    """uint8 / 255 -> conv 32 k8 s4, 64 k4 s2, 64 k3 s1 (VALID, relu) -> dense 256 relu -> softmax policy (A) + value (1);
    Keras Adam(LR, clipnorm=40, decay=5.12e-9): each gradient tensor clipped to norm 40 on its own."""
    config = globals()
    clipnorm = 40.0
    decay = 5.12e-9

    def build_arch(self):
        return archs.impala_keras_cnn(self.state_dim, self.action_dim)
