"""The diagonal Gaussian policy of PPO on top of the oracle (oracle/xt_oracle.py), for the tests of action_type
DiagGaussian.

The reference builds it in xt/model/ppo/ppo.py:62-95 and xt/model/tf_dist.py:49-86:
    log_std    = tf.get_variable('pi_logstd', shape=(1, A), initializer=zeros)     (created after the Keras model)
    dist_param = concat([pi_latent, pi_latent * 0.0 + log_std]);  std = exp(log_std)
    sample     = mean + std * N(0, 1);   log_prob(x) = -neglog_prob(x)
    neglog_prob(x) = 0.5 log(2 pi) A + 0.5 sum ((x - mean) / std)^2 + sum log_std
    entropy    = sum (log_std + 0.5 (log(2 pi) + 1))
and the clipped surrogate / value losses of xt/model/ppo/__init__.py:4-25 are unchanged.  A layer
("pi_logstd", "logstd", None, {"n": A}) holds the variable; every other layer goes through the oracle unchanged, in the
oracle's precision (orc.precision)."""
import math
from collections import OrderedDict

import numpy as np
import torch

from oracle import xt_oracle as orc

LOG_2PI = math.log(2.0 * math.pi)


def with_logstd(arch):
    """a PPO arch from the oracle with the pi_logstd layer appended, as archs.ppo_mlp / ppo_cnn(diag_gaussian=True)"""
    A = dict((n, sp) for n, _, _, sp in arch["layers"])["pi_latent"]["n"]
    return dict(arch, layers=list(arch["layers"]) + [("pi_logstd", "logstd", None, dict(n=A))])


def ppo_mlp_arch(**kw):
    return with_logstd(orc.ppo_mlp_arch(**kw))


def ppo_cnn_arch(**kw):
    return with_logstd(orc.ppo_cnn_arch(**kw))


def _base(arch):
    return dict(arch, layers=[l for l in arch["layers"] if l[1] != "logstd"])


def param_shapes(arch):
    out = orc.param_shapes(_base(arch))
    for name, kind, _, sp in arch["layers"]:
        if kind == "logstd":
            out[name] = (1, sp["n"])
    return out


def init_weights(arch, seed=0):
    """glorot_uniform kernels, zero biases and a zero pi_logstd"""
    w = orc.init_weights(_base(arch), seed=seed)
    for name, shape in param_shapes(arch).items():
        if name not in w:
            w[name] = np.zeros(shape, np.float32)
    return w


def forward(arch, weights, obs):
    """[mean (pi_latent), v]"""
    return orc.forward(_base(arch), {k: v for k, v in weights.items() if k != "pi_logstd"}, obs)


def _c(x, like):
    return torch.as_tensor(x, dtype=like.dtype)


def neglog_prob(x, mean, log_std):
    """tf_dist.py:63-66, [B, 1]; log_std broadcasts over the batch"""
    A = mean.shape[-1]
    return (_c(0.5 * LOG_2PI, mean) * A + 0.5 * (((x - mean) / torch.exp(log_std)) ** 2).sum(-1, keepdim=True)) + \
        log_std.expand_as(mean).sum(-1, keepdim=True)


def log_prob(x, mean, log_std):
    return -neglog_prob(x, mean, log_std)


def entropy(log_std):
    """tf_dist.py:71-72, [rows, 1]"""
    return (log_std + _c(0.5 * (LOG_2PI + 1.0), log_std)).sum(-1, keepdim=True)


def sample(mean, log_std, normals):
    """tf_dist.py:85-86 with the standard normals supplied"""
    return mean + torch.exp(log_std) * normals


def dist_log_std(mean, log_std):
    """the log_std half of dist_param: pi_latent * 0.0 + log_std (ppo.py:78) -- no gradient into pi_latent"""
    return mean * 0.0 + log_std


def ppo_gauss_loss(mean, log_std, v, action, old_logp, adv, old_v, target_v, clip_ratio, ent_coef, vf_clip, critic_coef):
    """actor_loss_with_entropy + critic_coef * critic_loss (xt/model/ppo/__init__.py:4-25, ppo.py:87-92); mean and action
    [B, A], log_std [1, A], the rest [B, 1]"""
    ls = dist_log_std(mean, log_std)
    logp = log_prob(action, mean, ls)
    ratio = torch.exp(logp - old_logp)
    s1 = ratio * adv
    s2 = torch.clamp(ratio, 1.0 - clip_ratio, 1.0 + clip_ratio) * adv
    actor = -torch.minimum(s1, s2).mean() - ent_coef * entropy(ls).mean()
    l1 = (v - target_v) ** 2
    vclip = old_v + torch.clamp(v - old_v, -vf_clip, vf_clip)
    critic = 0.5 * torch.maximum(l1, (vclip - target_v) ** 2).mean()
    return actor + critic_coef * critic


def predict(arch, weights, obs, normals):
    """PPO.predict (ppo.py:104-109) with supplied normals: (action [B, A], logp [B, 1], v [B, 1])"""
    with torch.no_grad():
        mean, v = forward(arch, weights, obs)
        ls = torch.from_numpy(np.asarray(weights["pi_logstd"])).to(mean.dtype)
        x = sample(mean, ls, torch.from_numpy(np.asarray(normals)).to(mean.dtype))
        return x.numpy(), log_prob(x, mean, ls).numpy(), v.numpy()


class PpoLearner(orc.PpoLearner):
    """orc.PpoLearner with the Gaussian head: pi_logstd is one more parameter (last, as TFVariables lists it) that
    counts toward the global-norm clip and takes Adam steps like the others; actions are float [N, A]."""

    def loss_and_grads(self, obs, action, old_logp, adv, old_v, target_v):
        w = dict(zip(self.names, self.params))
        mean, v = forward(self.arch, w, obs)
        f = orc._PREC["np"]
        tt = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=f)).view(-1, 1)   # noqa: E731
        act = torch.from_numpy(np.ascontiguousarray(action, dtype=f)).view(mean.shape)
        loss = ppo_gauss_loss(mean, w["pi_logstd"], v, act, tt(old_logp), tt(adv), tt(old_v), tt(target_v), self.cr, self.ec,
                              self.vfc, self.cc)
        return loss, torch.autograd.grad(loss, self.params)


def weights_in_order(arch, w):
    return OrderedDict((k, w[k]) for k in param_shapes(arch))
