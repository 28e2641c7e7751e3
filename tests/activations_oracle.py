"""The hidden activations of the reference's ACTIVATION_MAP (xt/model/model_utils.py:8-19) with TF 1.15's semantics, in
torch (any float dtype) and numpy float64, and the derivative rules the kernels use (gemm_f32.cuh act_grad).

install() adds them to the activation tables of the oracle (oracle/xt_oracle.py, oracle/np_f64.py), so its forward
passes and PPO learner run networks with these activations; relu, tanh and linear stay as the oracle defines them."""
import math

import numpy as np
import torch

LEAKY_ALPHA = 0.2                       # tf.nn.leaky_relu default
SELU_SCALE = 1.0507009873554805         # tf.nn.selu
SELU_ALPHA = 1.6732632423543772
GELU_C = math.sqrt(2.0 / math.pi)       # xt/model/tf_utils.py:157-166
GELU_A = 0.044715

NEW = ("sigmoid", "softsign", "softplus", "leaky_relu", "elu", "selu", "swish", "gelu")
KEEPS_Z = ("softsign", "swish", "gelu")     # the backward takes their derivative from the pre-activation z

TORCH = {
    "sigmoid": torch.sigmoid,
    "softsign": lambda x: x / (1 + x.abs()),
    "softplus": lambda x: torch.clamp(x, min=0) + torch.log1p(torch.exp(-x.abs())),
    "leaky_relu": lambda x: torch.where(x > 0, x, LEAKY_ALPHA * x),
    "elu": lambda x: torch.where(x > 0, x, torch.expm1(torch.clamp(x, max=0))),
    "selu": lambda x: SELU_SCALE * torch.where(x > 0, x, SELU_ALPHA * torch.expm1(torch.clamp(x, max=0))),
    "swish": lambda x: x * torch.sigmoid(x),
    "gelu": lambda x: 0.5 * x * (1 + torch.tanh(GELU_C * (x + GELU_A * x ** 3))),
}


def _np_sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


NUMPY = {
    "sigmoid": _np_sigmoid,
    "softsign": lambda x: x / (1 + np.abs(x)),
    "softplus": lambda x: np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x))),
    "leaky_relu": lambda x: np.where(x > 0, x, LEAKY_ALPHA * x),
    "elu": lambda x: np.where(x > 0, x, np.expm1(np.minimum(x, 0))),
    "selu": lambda x: SELU_SCALE * np.where(x > 0, x, SELU_ALPHA * np.expm1(np.minimum(x, 0))),
    "swish": lambda x: x * _np_sigmoid(x),
    "gelu": lambda x: 0.5 * x * (1 + np.tanh(GELU_C * (x + GELU_A * x ** 3))),
}


def grad_rule(act, y, z):
    """d act / d z as the kernels take it: from the output y, or from the pre-activation z for KEEPS_Z (numpy)."""
    if act == "sigmoid":
        return y * (1 - y)
    if act == "softsign":
        return 1.0 / (1 + np.abs(z)) ** 2
    if act == "softplus":
        return -np.expm1(-y)
    if act == "leaky_relu":
        return np.where(y > 0, 1.0, LEAKY_ALPHA)
    if act == "elu":
        return np.where(y > 0, 1.0, y + 1)
    if act == "selu":
        return np.where(y > 0, SELU_SCALE, y + SELU_SCALE * SELU_ALPHA)
    if act == "swish":
        s = _np_sigmoid(z)
        return s * (1 + z * (1 - s))
    if act == "gelu":
        t = np.tanh(GELU_C * (z + GELU_A * z ** 3))
        return 0.5 * (1 + t) + 0.5 * z * (1 - t * t) * GELU_C * (1 + 3 * GELU_A * z * z)
    raise KeyError(act)


def install():
    from oracle import np_f64
    from oracle import xt_oracle as orc
    for name in NEW:
        orc._ACT.setdefault(name, TORCH[name])
        np_f64._ACT.setdefault(name, NUMPY[name])
