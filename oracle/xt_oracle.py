"""CPU oracle for the xingtian actor-learner hot path.  TEST INFRASTRUCTURE ONLY.

This module is a *restatement* (numpy float64/float32 + torch-CPU fp32) of the
reference's numerics for the path SURVEY.md section 8 names.  It is imported
only by ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs -- never by ``xingtian_b200``.

PARITY STATUS: *partially pinned*.  The reference package cannot be imported
here as a whole (python 3.12 has no ``imp``; tensorflow==1.15 / gym / lz4 are
absent) and its tests hold no numeric golden vectors.  The pure-numpy pieces
of the reference (GAE ``data_proc``, the PPO minibatch loop, the DQN TD-target
loop, ``ReplayBuffer``, ``IMPALAOpt._data_proc``) ARE executed from
``/root/reference`` by ``tests/golden/make_golden.py`` (with stubbed TF
sessions) and this oracle is checked against those fixtures.  The reference's
loss code -- ``CategoricalDist`` (tf_dist.py:89-113), ``actor_loss_with_entropy``
/ ``critic_loss`` (model/ppo/__init__.py:4-25), ``vtrace.from_logic_outputs``
(impala/vtrace.py:39-115) and ``vtrace_loss`` (impala_cnn_opt.py:299-351) -- is
executed too, over a numpy stand-in for the dozen TensorFlow ops it calls
(``tf_losses.npz``): the STRUCTURE of those functions is pinned, the TF kernels
behind the individual ops are not.  What still bottoms out in tensorflow alone
(conv/dense layers, autodiff, ``AdamOptimizer``, ``clip_by_global_norm``,
``tf.random.categorical``, ``RMSPropOptimizer``, ``linear_cosine_decay``) is restated
from TF-1.15's documented semantics: for those rows parity against TensorFlow itself
is UNPINNED.  They are cross-checked independently instead (tests/test_oracle_f64.py):
conv/dense/flatten/SAME padding against a numpy-only float64 direct convolution
(oracle/np_f64.py, 1e-13), autograd against float64 finite differences, Adam /
RMSProp / the schedule against closed forms.  ``precision("f64")`` runs this module in
float64: the yardstick of the GPU parity tests.

Each function cites the reference file:line it follows (paths relative to
/root/reference).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from oracle.np_f64 import GELU_A, GELU_C, LEAKY_ALPHA, SELU_ALPHA, SELU_SCALE

# --------------------------------------------------------------------------- #
# Architectures
# --------------------------------------------------------------------------- #
# layer tuple: (name, kind, src, spec) ; kind in {"conv","dense","dueling","logstd"}
#   conv spec   : dict(k=, s=, cout=, pad="valid"|"same", act=)
#   dense spec  : dict(n=, act=)
#   dueling     : src = (value, adv), spec {}; the parameter-free Q = adv + (value - mean(value))
#   logstd spec : dict(n=A), src None; the (1, A) variable pi_logstd of the DiagGaussian head, no tensor
# tensors are named after the layer that produces them; the input is "obs".


def _ppo_heads(layers, tails, action_dim, diag_gaussian):
    layers.append(("pi_latent", "dense", tails.get("shared", tails.get("pi")), dict(n=action_dim, act=None)))
    layers.append(("output_value", "dense", tails.get("shared", tails.get("v")), dict(n=1, act=None)))
    if diag_gaussian:
        # tf.get_variable('pi_logstd', (1, A)) is created after the Keras model (xt/model/ppo/ppo.py:75-78), so it is
        # the last variable TFVariables lists
        layers.append(("pi_logstd", "logstd", None, dict(n=action_dim)))


def ppo_cnn_arch(state_dim=(84, 84, 4), action_dim=4, hidden_sizes=(256,),
                 activation="relu", vf_share_layers=True, diag_gaussian=False):
    """xt/model/model_utils.py:49-80 (get_cnn_backbone), :91-97, :120-162."""
    h, w, _ = state_dim
    if (h, w) == (84, 84):
        filt = [(32, 8, 4), (32, 4, 2), (64, 3, 1)]
    elif (h, w) == (42, 42):
        filt = [(32, 4, 2), (32, 4, 2), (64, 3, 1)]
    elif (h, w) == (15, 15):
        filt = [(32, 5, 1), (64, 3, 1), (64, 3, 1)]
    else:
        raise ValueError("no default filters for %r" % (state_dim,))
    layers = []
    prefixes = ["shared"] if vf_share_layers else ["pi", "v"]
    tails = {}
    for p in prefixes:
        src = "obs"
        for i, (co, k, s) in enumerate(filt):
            name = "%s_conv_layer_%d" % (p, i)
            layers.append((name, "conv", src, dict(k=k, s=s, cout=co, pad="valid", act=activation)))
            src = name
        for i, hs in enumerate(hidden_sizes):
            name = "%s_hidden_mlp_%d" % (p, i)
            layers.append((name, "dense", src, dict(n=hs, act=activation)))
            src = name
        tails[p] = src
    _ppo_heads(layers, tails, action_dim, diag_gaussian)
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0,
                layers=layers, outputs=["pi_latent", "output_value"])


def ppo_mlp_arch(state_dim=(4,), action_dim=2, hidden_sizes=(64, 64),
                 activation="tanh", vf_share_layers=False, diag_gaussian=False):
    """xt/model/model_utils.py:22-46 (get_mlp_backbone)."""
    layers = []
    prefixes = ["shared"] if vf_share_layers else ["pi", "v"]
    tails = {}
    for p in prefixes:
        src = "obs"
        for i, hs in enumerate(hidden_sizes):
            name = "%s_hidden_mlp_%d" % (p, i)
            layers.append((name, "dense", src, dict(n=hs, act=activation)))
            src = name
        tails[p] = src
    _ppo_heads(layers, tails, action_dim, diag_gaussian)
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0,
                layers=layers, outputs=["pi_latent", "output_value"])


def impala_cnn_arch(state_dim=(84, 84, 4), action_dim=4):
    """xt/model/impala/impala_cnn_opt.py:115-157; filters xt/model/atari_model.py:8-12."""
    h, w, _ = state_dim
    filt = [(16, 8, 4), (32, 4, 2), (256, 11, 1)] if (h, w) == (84, 84) else \
        [(16, 4, 2), (32, 4, 2), (256, 11, 1)]
    sc = "explore_agent/"
    layers = [
        (sc + "conv2d", "conv", "obs", dict(k=filt[0][1], s=filt[0][2], cout=filt[0][0], pad="same", act="relu")),
        (sc + "conv2d_1", "conv", sc + "conv2d", dict(k=filt[1][1], s=filt[1][2], cout=filt[1][0], pad="same", act="relu")),
        (sc + "conv2d_2", "conv", sc + "conv2d_1", dict(k=filt[2][1], s=filt[2][2], cout=filt[2][0], pad="valid", act="relu")),
        # 1x1 conv on a 1x1 map == dense on the flattened 256-vector
        (sc + "conv2d_3", "dense", sc + "conv2d_2", dict(n=action_dim, act=None)),
        (sc + "dense", "dense", sc + "conv2d_2", dict(n=1, act=None)),
    ]
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0,
                layers=layers, outputs=[sc + "conv2d_3", sc + "dense"])


def _dueling_head(layers, value, adv):
    """xt/model/dqn/dqn_cnn.py:53-58, dqn_mlp.py:50-54: adv = Dense(1) on the value head's input, then the combine."""
    layers.append((adv, "dense", layers[-1][2], dict(n=1, act=None)))
    layers.append(("dueling", "dueling", (value, adv), {}))
    return "dueling"


def dqn_cnn_arch(state_dim=(84, 84, 4), action_dim=4, dueling=False):
    """xt/model/dqn/dqn_cnn.py:45-58."""
    layers = [
        ("conv2d", "conv", "obs", dict(k=8, s=4, cout=32, pad="valid", act="relu")),
        ("conv2d_1", "conv", "conv2d", dict(k=4, s=2, cout=64, pad="valid", act="relu")),
        ("conv2d_2", "conv", "conv2d_1", dict(k=3, s=1, cout=64, pad="valid", act="relu")),
        ("dense", "dense", "conv2d_2", dict(n=256, act="relu")),
        ("dense_1", "dense", "dense", dict(n=action_dim, act=None)),
    ]
    out = _dueling_head(layers, "dense_1", "dense_2") if dueling else "dense_1"
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0,
                layers=layers, outputs=[out])


def dqn_mlp_arch(state_dim=(4,), action_dim=2, hidden_size=128, num_layers=1, dueling=False):
    """xt/model/dqn/dqn_mlp.py:43-60, :80-87."""
    layers = []
    src = "obs"
    for i in range(num_layers):
        name = "dense" if i == 0 else "dense_%d" % i
        layers.append((name, "dense", src, dict(n=hidden_size, act="relu")))
        src = name
    out = "dense_%d" % num_layers
    layers.append((out, "dense", src, dict(n=action_dim, act=None)))
    if dueling:
        out = _dueling_head(layers, out, "dense_%d" % (num_layers + 1))
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0,
                layers=layers, outputs=[out])


def _impala_keras_heads(trunk, action_dim):
    """output_actions = Dense(A, softmax), output_value = Dense(1) on the last hidden tensor (impala_mlp.py:49-50,
    impala_cnn.py:55-56); the softmax is applied by the loss and predict."""
    src = trunk[-1][0]
    return trunk + [("output_actions", "dense", src, dict(n=action_dim, act=None)),
                    ("output_value", "dense", src, dict(n=1, act=None))]


def impala_mlp_arch(state_dim=(4,), action_dim=2, hidden_size=128, num_layers=1):
    """ImpalaMlp, xt/model/impala/impala_mlp.py:39-50: DqnMlp's trunk, then the two heads."""
    trunk = dqn_mlp_arch(state_dim, action_dim, hidden_size, num_layers)["layers"][:num_layers]
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0,
                layers=_impala_keras_heads(trunk, action_dim), outputs=["output_actions", "output_value"])


def impala_keras_cnn_arch(state_dim=(84, 84, 4), action_dim=4):
    """ImpalaCnn (the Keras learner's model), xt/model/impala/impala_cnn.py:44-56: DqnCnn's trunk, then the two heads."""
    trunk = dqn_cnn_arch(state_dim, action_dim)["layers"][:4]
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0,
                layers=_impala_keras_heads(trunk, action_dim), outputs=["output_actions", "output_value"])


def _same_pad(size, k, s):
    """TF 'SAME': out=ceil(size/s); total=max((out-1)*s+k-size,0); before=total//2."""
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return out, total // 2, total - total // 2


def tensor_shapes(arch):
    """Shape (per sample) of every named tensor."""
    shapes = {"obs": tuple(arch["state_dim"])}
    for name, kind, src, sp in arch["layers"]:
        if kind == "logstd":
            continue
        if kind == "dueling":
            shapes[name] = shapes[src[0]]
            continue
        ish = shapes[src]
        if kind == "conv":
            h, w, _ = ish
            if sp["pad"] == "same":
                oh, ow = _same_pad(h, sp["k"], sp["s"])[0], _same_pad(w, sp["k"], sp["s"])[0]
            else:
                oh, ow = (h - sp["k"]) // sp["s"] + 1, (w - sp["k"]) // sp["s"] + 1
            shapes[name] = (oh, ow, sp["cout"])
        else:
            shapes[name] = (sp["n"],)
    return shapes


def param_shapes(arch):
    """OrderedDict{tf variable name -> shape}; conv kernels HWIO, dense [in,out].

    Names follow xt/model/model_utils.py:87,96 (layer names) + Keras' '/kernel',
    '/bias' suffixes, the key set TFVariables.get_weights returns
    (xt/model/tf_utils.py:99-102).  A dueling layer owns no variable; a logstd layer owns the (1, A) variable named
    after it."""
    shapes = tensor_shapes(arch)
    out = OrderedDict()
    for name, kind, src, sp in arch["layers"]:
        if kind == "dueling":
            continue
        if kind == "logstd":
            out[name] = (1, sp["n"])
            continue
        ish = shapes[src]
        if kind == "conv":
            out[name + "/kernel"] = (sp["k"], sp["k"], ish[-1], sp["cout"])
            out[name + "/bias"] = (sp["cout"],)
        else:
            out[name + "/kernel"] = (int(np.prod(ish)), sp["n"])
            out[name + "/bias"] = (sp["n"],)
    return out


def init_weights(arch, seed=0, baseline_norm_std=None):
    """Keras default init: glorot_uniform kernels, zero biases; pi_logstd starts at zero (xt/model/ppo/ppo.py:75-78)
    and draws nothing.

    ``baseline_norm_std`` restates custom_norm_initializer
    (xt/model/model_utils.py:204-211) for ImpalaCnnOpt's baseline dense."""
    rng = np.random.default_rng(seed)
    w = OrderedDict()
    for name, shp in param_shapes(arch).items():
        if not name.endswith("/kernel"):
            w[name] = np.zeros(shp, np.float32)
            continue
        if len(shp) == 4:
            rf = shp[0] * shp[1]
            fan_in, fan_out = rf * shp[2], rf * shp[3]
        else:
            fan_in, fan_out = shp
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        w[name] = rng.uniform(-lim, lim, size=shp).astype(np.float32)
        if baseline_norm_std is not None and name.endswith("explore_agent/dense/kernel"):
            o = rng.standard_normal(shp).astype(np.float32)
            o *= baseline_norm_std / np.sqrt(np.square(o).sum(axis=0, keepdims=True))
            w[name] = o.astype(np.float32)
    return w


_ACT = {
    None: lambda x: x, "linear": lambda x: x, "relu": torch.relu, "tanh": torch.tanh,
    # the rest of the reference's ACTIVATION_MAP, as np_f64 states them (any float dtype)
    "sigmoid": torch.sigmoid,
    "softsign": lambda x: x / (1 + x.abs()),
    "softplus": lambda x: torch.clamp(x, min=0) + torch.log1p(torch.exp(-x.abs())),
    "leaky_relu": lambda x: torch.where(x > 0, x, LEAKY_ALPHA * x),
    "elu": lambda x: torch.where(x > 0, x, torch.expm1(torch.clamp(x, max=0))),
    "selu": lambda x: SELU_SCALE * torch.where(x > 0, x, SELU_ALPHA * torch.expm1(torch.clamp(x, max=0))),
    "swish": lambda x: x * torch.sigmoid(x),
    "gelu": lambda x: 0.5 * x * (1 + torch.tanh(GELU_C * (x + GELU_A * x ** 3))),
}


# Arithmetic type of the network / loss / optimiser restatement.  fp32 is the reference's own precision (the golden
# fixtures and every bit-exact comparison use it); "f64" is the same code in float64: the error yardstick -- a parity
# test asserts |gpu - f64| <= 2 |torch-CPU fp32 - f64|, i.e. the CUDA path is as close to exact arithmetic as the
# reference's own fp32 execution is.
_PREC = {"t": torch.float32, "np": np.float32}


class precision(object):
    """with precision("f64"): ...   runs forward / learners / Adam in float64 (test-only yardstick)."""

    def __init__(self, name):
        self.new = {"f32": (torch.float32, np.float32), "f64": (torch.float64, np.float64)}[name]

    def __enter__(self):
        self.old = (_PREC["t"], _PREC["np"])
        _PREC["t"], _PREC["np"] = self.new
        return self

    def __exit__(self, *exc):
        _PREC["t"], _PREC["np"] = self.old
        return False


def dueling_combine(value, adv):
    """Q = adv + (value - mean over actions of value): the reference's arithmetic (xt/model/dqn/dqn_cnn.py:53-58,
    dqn_mlp.py:80-87)."""
    return adv + (value - value.mean(dim=1, keepdim=True))


def forward(arch, weights, obs, keep=False):
    """Network forward in torch-CPU fp32.  obs: ndarray/tensor [B,*state_dim].

    uint8 inputs are cast and divided by 255 (model_utils.py:187-189,
    dqn_cnn.py:48, state_transform :192-201 with mean 0).  Conv = NHWC,
    HWIO kernels (Keras Conv2D); flatten in HWC order (Keras Flatten on NHWC).
    A logstd layer produces no tensor; its variable is read by the Gaussian head."""
    wt = {k: (v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v))).to(_PREC["t"]) for k, v in weights.items()}
    x = obs if torch.is_tensor(obs) else torch.from_numpy(np.ascontiguousarray(obs))
    if arch["input_dtype"] == "uint8":
        x = x.to(_PREC["t"]) / 255.0
    else:
        x = x.to(_PREC["t"])
    t = {"obs": x}
    for name, kind, src, sp in arch["layers"]:
        if kind == "logstd":
            continue
        if kind == "dueling":
            t[name] = dueling_combine(t[src[0]], t[src[1]])
            continue
        a = t[src]
        if kind == "conv":
            xin = a.permute(0, 3, 1, 2)  # NCHW
            k = wt[name + "/kernel"].permute(3, 2, 0, 1)  # OIHW
            if sp["pad"] == "same":
                _, pt, pb = _same_pad(a.shape[1], sp["k"], sp["s"])
                _, pl, pr = _same_pad(a.shape[2], sp["k"], sp["s"])
                xin = F.pad(xin, (pl, pr, pt, pb))
            y = F.conv2d(xin, k, wt[name + "/bias"], stride=sp["s"])
            y = _ACT[sp["act"]](y).permute(0, 2, 3, 1)
        else:
            a2 = a.reshape(a.shape[0], -1)
            y = _ACT[sp["act"]](a2 @ wt[name + "/kernel"] + wt[name + "/bias"])
        t[name] = y
    if keep:
        return t
    return [t[o] for o in arch["outputs"]]


# --------------------------------------------------------------------------- #
# Categorical distribution / sampling
# --------------------------------------------------------------------------- #

def categorical_logp(logits, actions):
    """xt/model/tf_dist.py:103-106: -softmax_xent(one_hot(a), logits), shape [B,1]."""
    lsm = torch.log_softmax(logits, dim=-1)
    return lsm.gather(1, actions.long().view(-1, 1))


def categorical_entropy(logits):
    """xt/model/tf_dist.py:108-113, shape [B,1]."""
    r = logits - logits.max(dim=-1, keepdim=True).values
    e = torch.exp(r)
    z = e.sum(-1, keepdim=True)
    p = e / z
    return (p * (torch.log(z) - r)).sum(-1, keepdim=True)


def gumbel_argmax(logits, uniforms):
    """Shared-noise sampling contract: the form the reference keeps commented at
    xt/model/tf_dist.py:128-129 -- argmax(logits - log(-log(u))).  tf.random.categorical
    (tf_dist.py:130) draws from the same distribution with TF's own RNG stream, which
    cannot be reproduced; parity on action indices is therefore defined on supplied
    uniforms.  Computed in fp32 like the device path."""
    lg = np.asarray(logits, np.float32)
    u = np.asarray(uniforms, np.float32)
    g = -np.log(-np.log(u, dtype=np.float32), dtype=np.float32)
    return np.argmax(lg + g, axis=-1).astype(np.int32)


def philox4x32_10(counter, key):
    """Philox-4x32-10 (Salmon et al. 2011).  counter: uint32[...,4], key: uint32[2]."""
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
    c = [counter[..., i].astype(np.uint32) for i in range(4)]
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c[0].astype(np.uint64)
            p1 = M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), p0.astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), p1.astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0 = np.uint32(k0 + W0)
            k1 = np.uint32(k1 + W1)
    return np.stack(c, axis=-1)


def philox_uniforms(seed, offset, batch, adim):
    """Uniforms in (0,1) the device sampler draws when no noise tensor is supplied:
    sample b, action-group g (4 actions per Philox call) uses counter
    (b, g, offset_lo, offset_hi) and key (seed_lo, seed_hi);
    u = (x >> 8) * 2^-24 + 2^-25  (24-bit, never 0 or 1)."""
    groups = (adim + 3) // 4
    ctr = np.zeros((batch, groups, 4), np.uint32)
    ctr[..., 0] = np.arange(batch, dtype=np.uint32)[:, None]
    ctr[..., 1] = np.arange(groups, dtype=np.uint32)[None, :]
    ctr[..., 2] = np.uint32(offset & 0xFFFFFFFF)
    ctr[..., 3] = np.uint32((offset >> 32) & 0xFFFFFFFF)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    r = philox4x32_10(ctr, key).reshape(batch, groups * 4)[:, :adim]
    return ((r >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24) + np.float32(2.0 ** -25)).astype(np.float32)


def ppo_predict(arch, weights, obs, uniforms):
    """xt/model/ppo/ppo.py:104-109: (action[B] i32, logp[B,1], v[B,1]); logp of the
    sampled action (:85-86)."""
    with torch.no_grad():
        logits, v = forward(arch, weights, obs)
        act = gumbel_argmax(logits.numpy(), uniforms)
        logp = categorical_logp(logits, torch.from_numpy(act))
    return act, logp.numpy(), v.numpy()


# --------------------------------------------------------------------------- #
# DiagGaussian distribution (xt/model/tf_dist.py:49-86, xt/model/ppo/ppo.py:62-95)
# --------------------------------------------------------------------------- #
#   log_std    = tf.get_variable('pi_logstd', shape=(1, A), initializer=zeros)   (created after the Keras model)
#   dist_param = concat([pi_latent, pi_latent * 0.0 + log_std]);  std = exp(log_std)
#   sample     = mean + std * N(0, 1);   log_prob(x) = -neglog_prob(x)

LOG_2PI = math.log(2.0 * math.pi)


def _c(x, like):
    return torch.as_tensor(x, dtype=like.dtype)


def gauss_neglog_prob(x, mean, log_std):
    """tf_dist.py:63-66, [B, 1]; log_std broadcasts over the batch"""
    A = mean.shape[-1]
    return (_c(0.5 * LOG_2PI, mean) * A + 0.5 * (((x - mean) / torch.exp(log_std)) ** 2).sum(-1, keepdim=True)) + \
        log_std.expand_as(mean).sum(-1, keepdim=True)


def gauss_log_prob(x, mean, log_std):
    return -gauss_neglog_prob(x, mean, log_std)


def gauss_entropy(log_std):
    """tf_dist.py:71-72, [rows, 1]"""
    return (log_std + _c(0.5 * (LOG_2PI + 1.0), log_std)).sum(-1, keepdim=True)


def gauss_sample(mean, log_std, normals):
    """tf_dist.py:85-86 with the standard normals supplied"""
    return mean + torch.exp(log_std) * normals


def dist_log_std(mean, log_std):
    """the log_std half of dist_param: pi_latent * 0.0 + log_std (ppo.py:78) -- no gradient into pi_latent"""
    return mean * 0.0 + log_std


def ppo_gauss_predict(arch, weights, obs, normals):
    """PPO.predict (ppo.py:104-109) with supplied normals: (action [B, A], logp [B, 1], v [B, 1])"""
    with torch.no_grad():
        mean, v = forward(arch, weights, obs)
        ls = torch.from_numpy(np.asarray(weights["pi_logstd"])).to(mean.dtype)
        x = gauss_sample(mean, ls, torch.from_numpy(np.asarray(normals)).to(mean.dtype))
        return x.numpy(), gauss_log_prob(x, mean, ls).numpy(), v.numpy()


# --------------------------------------------------------------------------- #
# GAE  (agent side)
# --------------------------------------------------------------------------- #

GAMMA, LAM = 0.99, 0.95  # xt/agent/ppo/default_config.py:2-3


def gae(value, reward, done, gamma=GAMMA, lam=LAM):
    """xt/agent/ppo/ppo.py:77-106 (PPO.data_proc), one trajectory.

    value: [T+1,1] f32 (bootstrap appended, :73), reward: [T] (python floats =>
    float64 arithmetic), done: [T] bool.  Returns adv, old_value, target_value,
    each [T,1].  Arithmetic is float64 as in the reference (reward is f64, so
    numpy promotes); callers cast to f32 at the feed boundary."""
    value = np.asarray(value)
    next_value = value[1:]
    value = value[:-1]
    done = np.expand_dims(np.asarray(done, dtype=bool), axis=1)
    reward = np.expand_dims(np.asarray(reward, dtype=np.float64), axis=1)
    discount = ~done * gamma
    delta_t = reward + discount * next_value - value
    adv = delta_t
    for j in range(len(adv) - 2, -1, -1):
        adv[j] += adv[j + 1] * discount[j] * lam
    return adv, value, adv + value


def sign_clip_f32(reward):
    """np.sign of float32 rewards written as the device clips them: +-1, +0 for either zero, NaN kept"""
    r = np.asarray(reward, np.float32)
    one = np.float32(1)
    return np.where(r > 0, one, np.where(r < 0, -one, np.where(r == r, np.float32(0), r))).astype(np.float32)


def gae_f32(value, reward, done, gamma=GAMMA, lam=LAM, sign_clip=False):
    """gae's backward loop in plain float32 arithmetic, vectorised over rows: what fp32 rounding alone costs.

    value [..., T+1] (a trailing unit axis is dropped), reward / done [..., T]; gamma and lam are rounded to float32 as a
    C float argument carries them; sign_clip: rewards through sign_clip_f32 first.  Returns adv, old_value, target_value,
    each float32 [..., T]."""
    f = np.float32
    value = np.asarray(value, f)
    reward = np.asarray(reward, f)
    if value.shape[-1] == 1 and value.ndim == reward.ndim + 1:
        value = value[..., 0]
    if sign_clip:
        reward = sign_clip_f32(reward)
    done = np.asarray(done, bool)
    g, lm = f(gamma), f(lam)
    disc = np.where(done, f(0), g)
    delta = reward + disc * value[..., 1:] - value[..., :-1]
    adv = np.empty_like(delta)
    nxt = np.zeros(delta.shape[:-1], f)
    for t in range(delta.shape[-1] - 1, -1, -1):
        nxt = delta[..., t] + disc[..., t] * lm * nxt
        adv[..., t] = nxt
    return adv, value[..., :-1].copy(), adv + value[..., :-1]


def nstep_returns(reward, done, n, gamma, dtype=np.float64):
    """n-step returns of env-major segments [E, T] (or one segment [T]) in `dtype`, vectorised over rows: the window of
    step t stops after its first terminal step (inclusive), after n steps or at the end of the segment, m steps in all.
    Returns ret = sum_{k<m} gamma^k r_{t+k}, disc = gamma^m (0 when the window hit a terminal step), last = flat row index
    e * T + t + m - 1 (the row whose next state bootstraps) and done_n (the window hit a terminal step)."""
    f = np.dtype(dtype).type
    r = np.asarray(reward, f)
    d = np.asarray(done, bool)
    shape = r.shape
    r, d = r.reshape(-1, shape[-1]), d.reshape(-1, shape[-1])
    E, T = r.shape
    g = np.ones((E, T), f)
    acc = np.zeros((E, T), f)
    m = np.zeros((E, T), np.int64)
    term = np.zeros((E, T), bool)
    t = np.arange(T)
    for k in range(min(n, T)):
        live = ~term & (t + k < T)[None, :]          # windows still open at their k-th step
        rk = np.zeros((E, T), f)
        dk = np.zeros((E, T), bool)
        rk[:, :T - k], dk[:, :T - k] = r[:, k:], d[:, k:]
        acc = np.where(live, acc + g * rk, acc)
        g = np.where(live, g * f(gamma), g)
        m += live
        term |= live & dk
    last = np.arange(E)[:, None] * T + t[None, :] + m - 1
    return (acc.reshape(shape), np.where(term, f(0), g).reshape(shape), last.reshape(shape), term.reshape(shape))


# --------------------------------------------------------------------------- #
# PPO loss / optimiser / train loop
# --------------------------------------------------------------------------- #

def _surrogate(logp, old_logp, adv, clip_ratio):
    """the clipped surrogate, xt/model/ppo/__init__.py:4-11"""
    ratio = torch.exp(logp - old_logp)
    s1 = ratio * adv
    s2 = torch.clamp(ratio, 1.0 - clip_ratio, 1.0 + clip_ratio) * adv
    return torch.minimum(s1, s2).mean()


def _critic(v, old_v, target_v, vf_clip):
    """the clipped value loss, xt/model/ppo/__init__.py:17-25"""
    l1 = (v - target_v) ** 2
    vclip = old_v + torch.clamp(v - old_v, -vf_clip, vf_clip)
    l2 = (vclip - target_v) ** 2
    return 0.5 * torch.maximum(l1, l2).mean()


def ppo_loss(logits, v, action, old_logp, adv, old_v, target_v,
             clip_ratio, ent_coef, vf_clip, critic_coef):
    """xt/model/ppo/__init__.py:4-25 and xt/model/ppo/ppo.py:87-92.  All [B,1] but
    logits [B,A], action [B]."""
    surr = _surrogate(categorical_logp(logits, action), old_logp, adv, clip_ratio)
    ent = categorical_entropy(logits).mean()
    actor = -surr - ent_coef * ent
    return actor + critic_coef * _critic(v, old_v, target_v, vf_clip)


def ppo_gauss_loss(mean, log_std, v, action, old_logp, adv, old_v, target_v, clip_ratio, ent_coef, vf_clip, critic_coef):
    """ppo_loss with the DiagGaussian head; mean and action [B, A], log_std [1, A], the rest [B, 1]"""
    ls = dist_log_std(mean, log_std)
    actor = -_surrogate(gauss_log_prob(action, mean, ls), old_logp, adv, clip_ratio) - ent_coef * gauss_entropy(ls).mean()
    return actor + critic_coef * _critic(v, old_v, target_v, vf_clip)


def clip_by_global_norm(grads, clip):
    """tf.clip_by_global_norm: g * clip / max(||g||, clip)."""
    gn = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads))
    scale = clip / max(gn, clip)
    return [g * scale for g in grads], gn


def clip_per_tensor(grads, clipnorm):
    """Keras `clipnorm`: each gradient tensor g scaled by clipnorm / ||g|| where its norm exceeds clipnorm."""
    out = []
    for g in grads:
        n = float(g.double().pow(2).sum().sqrt())
        out.append(g * (clipnorm / n) if n > clipnorm else g)
    return out


class TFAdam:
    """tf.train.AdamOptimizer (xt/model/ppo/ppo.py:98; impala_cnn_opt.py:204):
    lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m,v EMA; theta -= lr_t*m/(sqrt(v)+eps)
    (the 'epsilon hat' form), eps=1e-8.  Keras Adam (dqn_cnn.py:60) uses the same
    update with eps=1e-7."""

    def __init__(self, params, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        self.params = params
        self.lr, self.b1, self.b2, self.eps = lr, beta1, beta2, eps
        self.m = [torch.zeros_like(p) for p in params]
        self.v = [torch.zeros_like(p) for p in params]
        self.f = _PREC["np"]
        self.b1p = self.f(1.0)
        self.b2p = self.f(1.0)

    def step(self, grads):
        f = self.f
        self.b1p = f(self.b1p * f(self.b1))
        self.b2p = f(self.b2p * f(self.b2))
        lr_t = f(self.lr) * np.sqrt(f(1) - self.b2p) / (f(1) - self.b1p)
        with torch.no_grad():
            for p, g, m, v in zip(self.params, grads, self.m, self.v):
                m.mul_(self.b1).add_(g, alpha=1 - self.b1)
                v.mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
                p.sub_(float(lr_t) * m / (v.sqrt() + self.eps))


class KerasAdam(TFAdam):
    """Keras (OptimizerV2) Adam, as documented for TF-1.15: the tf.train.Adam update with eps 1e-7, optional
    per-tensor clipnorm, and `decay`: lr / (1 + decay * iterations) with iterations counted before the step."""

    def __init__(self, params, lr, clipnorm=None, decay=0.0, eps=1e-7):
        super().__init__(params, lr, eps=eps)
        self.base_lr, self.clipnorm, self.decay, self.iterations = lr, clipnorm, decay, 0

    def step(self, grads):
        if self.clipnorm:
            grads = clip_per_tensor(grads, self.clipnorm)
        f = self.f
        self.lr = f(self.base_lr) / (f(1) + f(self.decay) * f(self.iterations)) if self.decay else self.base_lr
        self.iterations += 1
        super().step(grads)


class TFRMSProp:
    """tf.train.RMSPropOptimizer(lr, decay, epsilon, centered=True), momentum 0 (impala_cnn_opt.py:205-206), as documented
    for TF-1.15 (training_ops ApplyCenteredRMSProp): mg = rho mg + (1-rho) g; ms = rho ms + (1-rho) g^2;
    theta -= lr g / sqrt(ms - mg^2 + eps); the `rms` slot is initialised to ONES, `mg` to zeros."""

    def __init__(self, params, lr, decay=0.99, eps=0.1):
        self.params, self.lr, self.rho, self.eps = params, lr, decay, eps
        self.ms = [torch.ones_like(p) for p in params]
        self.mg = [torch.zeros_like(p) for p in params]

    def step(self, grads):
        with torch.no_grad():
            for p, g, ms, mg in zip(self.params, grads, self.ms, self.mg):
                mg.mul_(self.rho).add_(g, alpha=1 - self.rho)
                ms.mul_(self.rho).addcmul_(g, g, value=1 - self.rho)
                p.sub_(self.lr * g / (ms - mg * mg + self.eps).sqrt())


def linear_cosine_decay(lr, global_step, decay_steps, num_periods=0.5, alpha=0.0, beta=0.001):
    """tf.train.linear_cosine_decay as documented (used by impala_cnn_opt.py:234-249 with beta = schedule[1][1] / decay)."""
    s = min(float(global_step), float(decay_steps))
    linear = (decay_steps - s) / decay_steps
    cosine = 0.5 * (1.0 + math.cos(math.pi * 2.0 * num_periods * s / decay_steps))
    return lr * ((alpha + linear) * cosine + beta)


def _as_param_list(weights):
    return [torch.from_numpy(np.array(v, _PREC["np"], copy=True)).requires_grad_(True) for v in weights.values()]


class Learner:
    """What the learner restatements share: the arch, and the weights as leaf tensors of the working precision, in the
    order they were given."""

    def __init__(self, arch, weights):
        self.arch, self.names = arch, list(weights.keys())
        self.params = _as_param_list(weights)

    def named(self, params=None):
        return dict(zip(self.names, self.params if params is None else params))

    def weights(self):
        return OrderedDict((n, p.detach().numpy().copy()) for n, p in zip(self.names, self.params))


class PpoLearner(Learner):
    """Restates xt/model/ppo/ppo.py:62-132 (graph + train loop) on torch-CPU.  The action distribution follows the arch,
    as in the product: a logstd layer makes it DiagGaussian, its variable one more parameter (last, as TFVariables lists
    it) that counts toward the global-norm clip and takes Adam steps like the others; actions are then float [N, A]."""

    def __init__(self, arch, weights, lr=3e-4, batch_size=200, critic_coef=1.0, ent_coef=1e-3,
                 clip_ratio=0.2, max_grad_norm=5.0, num_sgd_iter=4, vf_clip=5.0):
        super().__init__(arch, weights)
        self.logstd = next((name for name, kind, _, _ in arch["layers"] if kind == "logstd"), None)
        self.opt = TFAdam(self.params, lr)
        self.bs, self.cc, self.ec, self.cr = batch_size, critic_coef, ent_coef, clip_ratio
        self.mgn, self.iters, self.vfc = max_grad_norm, num_sgd_iter, vf_clip
        self.last_grad_norm = None

    def loss_and_grads(self, obs, action, old_logp, adv, old_v, target_v):
        w = self.named()
        head, v = forward(self.arch, w, obs)
        f = _PREC["np"]
        tt = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=f)).view(-1, 1)   # noqa: E731
        hp = (self.cr, self.ec, self.vfc, self.cc)
        if self.logstd is None:
            loss = ppo_loss(head, v, torch.from_numpy(np.ascontiguousarray(action)), tt(old_logp), tt(adv),
                            tt(old_v), tt(target_v), *hp)
        else:
            act = torch.from_numpy(np.ascontiguousarray(action, dtype=f)).view(head.shape)
            loss = ppo_gauss_loss(head, w[self.logstd], v, act, tt(old_logp), tt(adv), tt(old_v), tt(target_v), *hp)
        grads = torch.autograd.grad(loss, self.params)
        return loss, grads

    def sgd_step(self, obs, action, old_logp, adv, old_v, target_v):
        loss, grads = self.loss_and_grads(obs, action, old_logp, adv, old_v, target_v)
        grads, gn = clip_by_global_norm(grads, self.mgn)
        self.last_grad_norm = gn
        self.opt.step(grads)
        return float(loss.detach())

    def train(self, state, label, rng=np.random):
        """xt/model/ppo/ppo.py:111-132.  `inds` is shuffled IN PLACE every epoch
        (cumulative permutation), ragged last minibatch kept."""
        nbatch = state[0].shape[0]
        inds = np.arange(nbatch)
        loss_val = []
        for _ in range(self.iters):
            rng.shuffle(inds)
            for start in range(0, nbatch, self.bs):
                mb = inds[start:start + self.bs]
                loss_val.append(self.sgd_step(state[0][mb], label[0][mb], label[1][mb], label[2][mb],
                                              label[3][mb], label[4][mb]))
        return float(np.mean(loss_val)), loss_val


# --------------------------------------------------------------------------- #
# IMPALA: V-trace + loss
# --------------------------------------------------------------------------- #

def vtrace_from_logits(bp_logits, tp_logits, actions, discounts, rewards, values, bootstrap,
                       clip_rho=1.0, clip_pg_rho=1.0):
    """xt/model/impala/vtrace.py:39-115.  Inputs time-major [T,B,(A)] numpy, computed in the working precision:
    logits are cast to it, the other inputs widened to at least it.  Returns vs[T,B], pg_adv[T,B]."""
    f = _PREC["np"]

    def logp(lg, a):
        m = lg.max(-1, keepdims=True)
        lse = m + np.log(np.exp(lg - m).sum(-1, keepdims=True))
        return np.take_along_axis(lg - lse, a[..., None].astype(np.int64), -1)[..., 0]

    def widen(x):
        x = np.asarray(x)
        return x.astype(np.promote_types(x.dtype, f), copy=False)

    discounts, rewards, values, bootstrap = widen(discounts), widen(rewards), widen(values), widen(bootstrap)
    tlp = logp(tp_logits.astype(f), actions)
    blp = logp(bp_logits.astype(f), actions)
    rho = np.exp(tlp - blp).astype(f)
    crho = np.minimum(f(clip_rho), rho)
    cpg = np.minimum(f(clip_pg_rho), rho)
    cs = np.minimum(f(1.0), rho)
    nv = np.concatenate([values[1:], bootstrap[None]], 0)
    deltas = crho * (rewards + discounts * nv - values)
    acc = np.zeros_like(bootstrap, dtype=f)
    out = np.zeros_like(values, dtype=f)
    for t in range(values.shape[0] - 1, -1, -1):
        acc = (deltas[t] + discounts[t] * cs[t] * acc).astype(f)
        out[t] = acc
    vs = out + values
    vs_next = np.concatenate([vs[1:], bootstrap[None]], 0)
    pg = cpg * (rewards + discounts * vs_next - values)
    return vs.astype(f), pg.astype(f)


def split_batches(x, batch_step, drop_last=False):
    """impala_cnn_opt.py:171-186: [count*step, ...] -> [step, count, ...]."""
    count = x.shape[0] // batch_step
    r = x.reshape((count, batch_step) + tuple(x.shape[1:]))
    r = r.transpose(0, 1) if torch.is_tensor(r) else np.swapaxes(r, 0, 1)
    return r[:-1] if drop_last else r


def impala_loss(tp_logits_flat, baseline_flat, bp_logits, actions, dones, rewards, batch_step, gamma=0.99):
    """impala_cnn_opt.py:188-196 + :299-351.  tp_logits_flat [N,A] / baseline_flat [N]
    torch tensors (grad flows); the rest numpy, env-major flat [N].  The V-trace targets are computed in the working
    precision."""
    f = _PREC["np"]
    tp = split_batches(tp_logits_flat, batch_step, True)
    val = split_batches(baseline_flat, batch_step, True)
    boot = split_batches(baseline_flat, batch_step)[-1]
    bp = split_batches(np.asarray(bp_logits, f), batch_step, True)
    act = split_batches(np.asarray(actions, np.int32), batch_step, True)
    disc = split_batches((~np.asarray(dones, bool)).astype(f) * f(gamma), batch_step, True)
    rew = split_batches(np.clip(np.asarray(rewards, f), -1, 1), batch_step, True)
    vs, pg = vtrace_from_logits(bp, tp.detach().numpy(), act, disc, rew, val.detach().numpy(), boot.detach().numpy())
    vs_t, pg_t = torch.from_numpy(vs).to(_PREC["t"]), torch.from_numpy(pg).to(_PREC["t"])
    lsm = torch.log_softmax(tp, -1)
    xent = -lsm.gather(-1, torch.from_numpy(act.astype(np.int64))[..., None])[..., 0]
    pi_loss = (xent * pg_t).sum()
    val_loss = 0.5 * ((vs_t - val) ** 2).sum()
    ent_loss = -(-(torch.softmax(tp, -1) * lsm).sum(-1)).sum()
    return pi_loss + 0.5 * val_loss + 0.01 * ent_loss


class ImpalaLearner(Learner):
    """Restates ImpalaCnnOpt's train graph (impala_cnn_opt.py:188-217, :251-265)."""

    def __init__(self, arch, weights, lr=0.0005, grad_norm_clip=40.0, sample_batch_step=128, gamma=0.99, opt_type="adam",
                 lr_schedule=None):
        super().__init__(arch, weights)
        self.opt = TFAdam(self.params, lr) if opt_type == "adam" else TFRMSProp(self.params, lr)
        self.lr_schedule, self.global_step = (lr_schedule if opt_type == "adam" else None), 0
        self.clip, self.step_len, self.gamma = grad_norm_clip, sample_batch_step, gamma
        self.last_grad_norm = None

    def loss_and_grads(self, state, bp_logits, actions, dones, rewards):
        logits, base = forward(self.arch, self.named(), state)
        loss = impala_loss(logits, base[:, 0], bp_logits, actions, dones, rewards, self.step_len, self.gamma)
        return loss, torch.autograd.grad(loss, self.params)

    def train(self, state, label):
        loss, grads = self.loss_and_grads(state, *label)
        grads, gn = clip_by_global_norm(grads, self.clip)
        self.last_grad_norm = gn
        if self.lr_schedule:
            self.opt.lr = linear_cosine_decay(self.lr_schedule[0][1], self.global_step, 20000.0, beta=self.lr_schedule[1][1] / 20000.0)
        self.global_step += 1
        self.opt.step(grads)
        return float(loss.detach())


# --------------------------------------------------------------------------- #
# DQN
# --------------------------------------------------------------------------- #

def dqn_targets(y_online, target_q, actions, rewards, dones, gamma=0.99, q_next_online=None, disc=None):
    """xt/algorithm/dqn/dqn.py:79-95: 1-step TD target written into y[k,a_k], y in float32.
    Double-DQN when q_next_online is given (:79-84), the first maximum of its row winning.  `disc` holds a per-row
    discount (an n-step target, as xtb_dqn_td_loss_grad takes it) that replaces gamma; y then keeps the precision of
    y_online.  Under precision("f64") y and every input it is built from are float64."""
    if _PREC["np"] is np.float64:
        y_online, target_q, rewards = (np.asarray(x, np.float64) for x in (y_online, target_q, rewards))
        disc = None if disc is None else np.asarray(disc, np.float64)
        y = np.array(y_online, copy=True)
    else:
        y = np.array(y_online, np.float32 if disc is None else None, copy=True)
    best = np.argmax(q_next_online if q_next_online is not None else target_q, 1)
    maxq = target_q[np.arange(len(y)), best]
    for k in range(len(y)):
        y[k][actions[k]] = rewards[k] if dones[k] else rewards[k] + (gamma if disc is None else disc[k]) * maxq[k]
    return y


class DqnLearner(Learner):
    """Restates DQN.train (xt/algorithm/dqn/dqn.py:61-103) + Keras compile(mse,
    Adam(clipnorm=10)) (xt/model/dqn/dqn_cnn.py:60-61): mse = mean over B*A;
    clipnorm clips EACH gradient tensor to norm<=10; Adam eps=1e-7.  `disc` / `huber` extend the TD target and
    loss the way xtb_dqn_td_loss_grad does: a per-row discount, and Huber with that delta; `weights` scale each row's
    loss (Keras sample_weight).  The target net starts as a copy of the online weights, or from `target_weights`."""

    def __init__(self, arch, weights, lr=0.00015, clipnorm=10.0, gamma=0.99, target_update_freq=1000,
                 double_dqn=False, target_weights=None):
        super().__init__(arch, weights)
        self.target = [p.detach().clone() for p in self.params] if target_weights is None else \
            [p.detach() for p in _as_param_list(OrderedDict((n, target_weights[n]) for n in self.names))]
        self.opt = TFAdam(self.params, lr, eps=1e-7)
        self.clipnorm, self.gamma, self.freq, self.double = clipnorm, gamma, target_update_freq, double_dqn
        self.train_count = 0

    def predict(self, states, target=False):
        with torch.no_grad():
            return forward(self.arch, self.named(self.target if target else None), states)[0].numpy()

    def loss_and_grads(self, states, actions, rewards, new_states, dones, disc=None, huber=0.0, weights=None):
        """the loss 1/(B A) sum_b w_b sum_a e_ba, its gradients, the targets y [B, A] and |y - Q(s, a)| [B]"""
        y_t = self.predict(states)
        tq = self.predict(new_states, target=True)
        qn = self.predict(new_states) if self.double else None
        y = dqn_targets(y_t, tq, actions, rewards, dones, self.gamma, qn, disc)
        q = forward(self.arch, self.named(), states)[0]
        diff = q - torch.from_numpy(y)
        if huber > 0:
            ad = diff.abs()
            per = torch.where(ad <= huber, 0.5 * diff * diff, huber * (ad - 0.5 * huber))
        else:
            per = diff * diff
        if weights is not None:
            per = per * torch.from_numpy(np.asarray(weights)).to(per.dtype)[:, None]
        loss = per.mean()
        td_abs = diff.detach().abs().numpy()[np.arange(len(y)), np.asarray(actions, np.int64)]
        return loss, torch.autograd.grad(loss, self.params), y, td_abs

    def train(self, states, actions, rewards, new_states, dones, disc=None, huber=0.0):
        loss, grads, _, _ = self.loss_and_grads(states, actions, rewards, new_states, dones, disc, huber)
        if self.clipnorm:
            grads = clip_per_tensor(grads, self.clipnorm)
        self.opt.step(grads)
        self.train_count += 1
        if self.train_count % self.freq == 0:
            self.target = [p.detach().clone() for p in self.params]
        return float(loss.detach())


# --------------------------------------------------------------------------- #
# Synthetic rollouts (SURVEY.md section 8(d))
# --------------------------------------------------------------------------- #

def synth_ppo_rollout(seed, env_num, steps, state_dim=(84, 84, 4), action_dim=4, dtype=np.uint8):
    """Seeded synthetic rollout, env-major [E*T,...]."""
    rng = np.random.default_rng(seed)
    n = env_num * steps
    if dtype == np.uint8:
        obs = rng.integers(0, 256, size=(n,) + tuple(state_dim), dtype=np.uint8)
    else:
        obs = rng.standard_normal((n,) + tuple(state_dim)).astype(np.float32)
    action = rng.integers(0, action_dim, size=n).astype(np.int32)
    reward = rng.choice(np.array([-1.0, 0.0, 1.0]), size=n, p=[0.05, 0.9, 0.05])
    done = rng.random(n) < (1.0 / 200.0)
    value = rng.standard_normal((env_num, steps + 1, 1)).astype(np.float32)
    logits = rng.standard_normal((n, action_dim)).astype(np.float32)
    lsm = logits - np.log(np.exp(logits).sum(-1, keepdims=True))
    logp = np.take_along_axis(lsm, action[:, None].astype(np.int64), 1).astype(np.float32)
    return dict(obs=obs, action=action, reward=reward, done=done, value=value, logp=logp, logits=logits)
