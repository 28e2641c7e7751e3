"""TEST INFRASTRUCTURE -- float64 numpy restatement of the network forward, independent of torch.

Purpose (round-1 verdict, row c "nothing independent checks the TF-bottomed ops"): the torch-CPU oracle in
xt_oracle.py restates Keras Conv2D / Dense / Flatten from their documentation with torch ops.  This module computes the
same forward with nothing but numpy indexing and a tensordot, in float64, so the two restatements pin each other
(tests/test_oracle_f64.py) and the float64 result is the exact-arithmetic yardstick of the GPU parity tests.

Follows xt/model/model_utils.py:141-160 (Conv2D NHWC, HWIO kernels, 'valid' / 'same' padding as TensorFlow defines it:
pad_total = max((ceil(in/s)-1)*s + k - in, 0), the smaller half first), :187-201 (uint8 -> /255), Keras Flatten
(row-major over H, W, C) and Dense (x @ kernel + bias).

It also holds the hidden activations of the reference's ACTIVATION_MAP (xt/model/model_utils.py:8-19) with TF 1.15's
semantics, their constants and the derivative rules the kernels use (gemm_f32.cuh act_grad); xt_oracle takes the
constants from here.
"""
import math

import numpy as np


def _same_pad(size, k, s):
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def conv2d_nhwc(x, kernel, bias, stride, pad):
    """x [B,H,W,C] float64, kernel [kh,kw,C,O], bias [O]; returns [B,OH,OW,O]."""
    kh, kw, c, o = kernel.shape
    if pad == "same":
        pt, pb = _same_pad(x.shape[1], kh, stride)
        pl, pr = _same_pad(x.shape[2], kw, stride)
        x = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    b, h, w, _ = x.shape
    oh, ow = (h - kh) // stride + 1, (w - kw) // stride + 1
    out = np.zeros((b, oh, ow, o), np.float64)
    for ky in range(kh):                      # direct form: one shifted strided view per tap
        for kx in range(kw):
            patch = x[:, ky:ky + (oh - 1) * stride + 1:stride, kx:kx + (ow - 1) * stride + 1:stride, :]
            out += np.tensordot(patch, kernel[ky, kx], axes=([3], [0]))
    return out + bias


LEAKY_ALPHA = 0.2                       # tf.nn.leaky_relu default
SELU_SCALE = 1.0507009873554805         # tf.nn.selu
SELU_ALPHA = 1.6732632423543772
GELU_C = math.sqrt(2.0 / math.pi)       # xt/model/tf_utils.py:157-166
GELU_A = 0.044715

NEW = ("sigmoid", "softsign", "softplus", "leaky_relu", "elu", "selu", "swish", "gelu")   # past relu / tanh
KEEPS_Z = ("softsign", "swish", "gelu")     # the backward takes their derivative from the pre-activation z


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


_ACT = {
    None: lambda v: v, "linear": lambda v: v, "relu": lambda v: np.maximum(v, 0.0), "tanh": np.tanh,
    "sigmoid": _sigmoid,
    "softsign": lambda x: x / (1 + np.abs(x)),
    "softplus": lambda x: np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x))),
    "leaky_relu": lambda x: np.where(x > 0, x, LEAKY_ALPHA * x),
    "elu": lambda x: np.where(x > 0, x, np.expm1(np.minimum(x, 0))),
    "selu": lambda x: SELU_SCALE * np.where(x > 0, x, SELU_ALPHA * np.expm1(np.minimum(x, 0))),
    "swish": lambda x: x * _sigmoid(x),
    "gelu": lambda x: 0.5 * x * (1 + np.tanh(GELU_C * (x + GELU_A * x ** 3))),
}


def grad_rule(act, y, z):
    """d act / d z as the kernels take it: from the output y, or from the pre-activation z for KEEPS_Z."""
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
        s = _sigmoid(z)
        return s * (1 + z * (1 - s))
    if act == "gelu":
        t = np.tanh(GELU_C * (z + GELU_A * z ** 3))
        return 0.5 * (1 + t) + 0.5 * z * (1 - t * t) * GELU_C * (1 + 3 * GELU_A * z * z)
    raise KeyError(act)


def forward(arch, weights, obs):
    """dict name -> float64 activations of every layer (same arch dicts as xt_oracle); a logstd layer holds a variable
    and produces no tensor."""
    x = np.asarray(obs).astype(np.float64)
    if arch["input_dtype"] == "uint8":
        x = x / 255.0
    t = {"obs": x}
    for name, kind, src, sp in arch["layers"]:
        if kind == "logstd":
            continue
        if kind == "dueling":
            value, adv = t[src[0]], t[src[1]]
            t[name] = adv + (value - value.mean(1, keepdims=True))
            continue
        a = t[src]
        k = np.asarray(weights[name + "/kernel"], np.float64)
        b = np.asarray(weights[name + "/bias"], np.float64)
        if kind == "conv":
            y = conv2d_nhwc(a, k, b, sp["s"], sp["pad"])
        else:
            y = a.reshape(a.shape[0], -1) @ k + b
        t[name] = _ACT[sp["act"]](y)
    return t


def adam_steps(p0, grads, lr, b1=0.9, b2=0.999, eps=1e-8):
    """tf.train.AdamOptimizer in float64 on a flat vector: lr_t = lr*sqrt(1-b2^t)/(1-b1^t); p -= lr_t*m/(sqrt(v)+eps)."""
    p = np.array(p0, np.float64)
    m = np.zeros_like(p); v = np.zeros_like(p)
    for t, g in enumerate(grads, 1):
        g = np.asarray(g, np.float64)
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        p = p - lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t) * m / (np.sqrt(v) + eps)
    return p
