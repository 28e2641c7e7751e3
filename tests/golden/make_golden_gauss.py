#!/usr/bin/env python
"""Generate ppo_gauss.npz by EXECUTING the reference's own diagonal Gaussian distribution and PPO losses:

    DiagGaussianDist (xt/model/tf_dist.py:49-86, with the log_prob it inherits from ActionDist)
    actor_loss_with_entropy, critic_loss (xt/model/ppo/__init__.py:4-25)

over make_golden.TFShim (eager float32), which gains the ops these functions use: tf.split, tf.shape, tf.cast and
tf.random_normal, the last fed from supplied standard normals.  The distribution parameter is built as PPO.build_graph
builds it for DiagGaussian (xt/model/ppo/ppo.py:75-78): concat([pi_latent, pi_latent * 0.0 + log_std]).

For A in 1, 3, 6: seeded pi_latent [B, A], log_std [1, A], normals [B, A]; recorded are the samples and their log_prob,
neglog_prob and entropy, and for behaviour actions drawn from a perturbed policy the actor, critic and total losses
(total = actor + CRITIC_LOSS_COEF * critic, ppo.py:87-92).

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_gauss.py
It writes ppo_gauss.npz alone; the other fixtures are untouched."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

B = 64
CLIP, ENT, VF_CLIP, CRITIC_COEF = 0.2, 0.01, 5.0, 1.0


class _TFTensor(np.ndarray):
    """A float32 tensor: a numpy float64 constant multiplied into it is converted to float32 first, as TF converts
    `0.5 * np.log(2.0 * np.pi) * tensor` (tf_dist.py:64), instead of numpy promoting the product to float64."""

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        args = [np.asarray(x.view(np.ndarray) if isinstance(x, _TFTensor) else x, np.float32) for x in inputs]
        return getattr(ufunc, method)(*args, **kwargs)


class GaussTFShim(mg.TFShim):
    normals = None     # what the next tf.random_normal returns

    @staticmethod
    def split(x, num_or_size_splits, axis=-1):
        return np.split(np.asarray(x, np.float32), num_or_size_splits, axis=axis)

    @staticmethod
    def shape(x):
        return np.asarray(np.shape(x), np.int32)

    @staticmethod
    def cast(x, dtype):
        return np.asarray(np.asarray(x).astype(dtype)).view(_TFTensor)

    @staticmethod
    def random_normal(shape, dtype=None):
        n = np.asarray(GaussTFShim.normals, np.float32)
        assert tuple(n.shape) == tuple(int(s) for s in shape), (n.shape, shape)
        return n


def reference_modules():
    mg.install_stubs()
    compat = mg._AnyName("xt.model.tf_compat")
    compat.tf = GaussTFShim
    sys.modules["xt.model.tf_compat"] = compat
    dist_mod = mg._load("xt.model.tf_dist", "xt/model/tf_dist.py")
    ppo_mod = mg._load("xt.model.ppo", "xt/model/ppo/__init__.py")
    return dist_mod, ppo_mod


def golden_gauss():
    dist_mod, ppo_mod = reference_modules()
    tf = GaussTFShim
    rng = np.random.default_rng(4242)
    out = {}
    for A in (1, 3, 6):
        pre = "A%d_" % A
        mean = (rng.standard_normal((B, A)) * 0.8).astype(np.float32)
        log_std = (rng.standard_normal((1, A)) * 0.4).astype(np.float32)
        normals = rng.standard_normal((B, A)).astype(np.float32)
        dist = dist_mod.DiagGaussianDist(A)
        dist.init_by_param(tf.concat([mean, mean * 0.0 + log_std], axis=-1))
        GaussTFShim.normals = normals
        sample = dist.sample()
        # behaviour actions of a perturbed policy; its log-probabilities spread the ratio over both sides of the clip
        behav = (mean + 0.3 * rng.standard_normal((B, A)) + np.exp(log_std) * rng.standard_normal((B, A)) * 1.2).astype(np.float32)
        old_logp = (dist.log_prob(behav) + 0.4 * rng.standard_normal((B, 1))).astype(np.float32)
        adv = rng.standard_normal((B, 1)).astype(np.float32)
        old_v, target_v = rng.standard_normal((B, 1)).astype(np.float32), rng.standard_normal((B, 1)).astype(np.float32)
        out_v = (old_v + 4.0 * rng.standard_normal((B, 1))).astype(np.float32)
        actor = np.float32(ppo_mod.actor_loss_with_entropy(dist, adv, old_logp, behav, CLIP, ENT))
        critic = np.float32(ppo_mod.critic_loss(target_v, out_v, old_v, VF_CLIP))
        arrays = dict(mean=mean, log_std=log_std, normals=normals, sample=sample, sample_logp=dist.log_prob(sample),
                      behav=behav, behav_neglogp=dist.neglog_prob(behav), entropy=dist.entropy(), old_logp=old_logp,
                      adv=adv, old_v=old_v, target_v=target_v, out_v=out_v, actor_loss=actor, critic_loss=critic,
                      total_loss=np.float32(actor + np.float32(CRITIC_COEF) * critic))
        out.update({pre + k: np.asarray(v) for k, v in arrays.items()})
    out["hyper"] = np.asarray([CLIP, ENT, VF_CLIP, CRITIC_COEF], np.float32)
    np.savez(os.path.join(HERE, "ppo_gauss.npz"), **out)
    print("ppo_gauss.npz", {A: float(out["A%d_total_loss" % A]) for A in (1, 3, 6)})


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        sys.exit("needs /root/reference")
    golden_gauss()
