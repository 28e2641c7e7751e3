"""CPU oracle for IMPALA with the Keras learner (xt/algorithm/impala/impala.py, xt/model/impala/impala_mlp.py and
impala_cnn.py), on top of oracle/xt_oracle.py.  TEST INFRASTRUCTURE ONLY.

Pinned by tests/golden/impala_keras.npz (the reference's own _train_proc / train slicing and impala_loss closures,
executed by tests/golden/make_golden_impala_keras.py): the V-trace variant, the slices, the loss value.  Restated from
documented TF-1.15 behaviour and unpinned, like tf.train.AdamOptimizer in xt_oracle:
  * training_arrays.fit_loop: one np.random.shuffle(np.arange(n)) per fit call, consecutive batches of 128, the last
    one ragged;
  * OptimizerV2 `decay`: lr / (1 + decay * iterations), iterations counted before the step; clipnorm per tensor;
  * the epoch loss fit reports: per-batch losses weighted by batch size, i.e. sum over rows of the row loss / n."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import xt_oracle as orc

FIT_BATCH = 128


def _dense(name, src, n, act):
    return (name, "dense", src, dict(n=n, act=act))


def impala_mlp_arch(state_dim=(4,), action_dim=2, hidden_size=128, num_layers=1):
    """impala_mlp.py:39-50 (the softmax of output_actions is applied by the loss / predict below)."""
    layers, src = [], "obs"
    for i in range(num_layers):
        name = "dense" if i == 0 else "dense_%d" % i
        layers.append(_dense(name, src, hidden_size, "relu"))
        src = name
    layers += [_dense("output_actions", src, action_dim, None), _dense("output_value", src, 1, None)]
    return dict(input_dtype="float32", state_dim=tuple(state_dim), scale=1.0, layers=layers,
                outputs=["output_actions", "output_value"])


def impala_cnn_arch(state_dim=(84, 84, 4), action_dim=4):
    """impala_cnn.py:44-56."""
    layers = [("conv2d", "conv", "obs", dict(k=8, s=4, cout=32, pad="valid", act="relu")),
              ("conv2d_1", "conv", "conv2d", dict(k=4, s=2, cout=64, pad="valid", act="relu")),
              ("conv2d_2", "conv", "conv2d_1", dict(k=3, s=1, cout=64, pad="valid", act="relu")),
              _dense("dense", "conv2d_2", 256, "relu"),
              _dense("output_actions", "dense", action_dim, None), _dense("output_value", "dense", 1, None)]
    return dict(input_dtype="uint8", state_dim=tuple(state_dim), scale=1.0 / 255.0, layers=layers,
                outputs=["output_actions", "output_value"])


# --------------------------------------------------------------------------------------------------------- V-trace
def vtrace(probs, values, behav, amat, reward, done, gamma=0.99):
    """IMPALA._train_proc (impala.py:124-184) in float64.  probs [n, L+1, A] / values [n, L+1] of the target network
    over every state, behav / amat [n, L, A], reward / done [n, L].  Returns pg_adv, target_value flat [n*L]."""
    f = np.float64
    probs, values = np.asarray(probs, f), np.asarray(values, f)
    behav, amat, reward = np.asarray(behav, f), np.asarray(amat, f), np.asarray(reward, f)
    disc = (~np.asarray(done, bool)) * gamma
    logp = lambda p: np.log((p * amat).sum(-1) + 1e-10)   # noqa: E731
    rho = np.minimum(np.exp(logp(probs[:, :-1]) - logp(behav)), 1.0)
    v, vn = values[:, :-1], values[:, 1:]
    adv = rho * (reward + disc * vn - v)
    L = adv.shape[1]
    for j in range(L - 2, -1, -1):
        adv[:, j] += adv[:, j + 1] * disc[:, j + 1] * rho[:, j + 1]
    tv = v + adv
    tv_next = np.concatenate([tv[:, 1:], vn[:, -1:]], 1)
    pg = rho * (reward + disc * tv_next - v)
    return pg.reshape(-1), tv.reshape(-1)


# --------------------------------------------------------------------------------------------------------- loss
def row_losses(logits, value, y, adv, tv, ent=0.01):
    """Per-row Keras loss: impala_loss (impala_mlp.py:82-93) on softmax(logits) + 0.5 * mse(value), torch tensors
    (autograd flows through log(p + 1e-10) and the softmax)."""
    p = torch.softmax(logits, -1)
    lp = torch.log(p + 1e-10)
    pol = (adv.reshape(-1, 1) * (-y * lp) - ent * (-p * lp)).mean(-1)
    return pol + 0.5 * (value.reshape(-1) - tv.reshape(-1)) ** 2


def impala_loss_value(probs, y, adv, ent=0.01):
    """The impala_loss closure's value on given probabilities (for the golden fixture): mean over rows and actions."""
    p, y, adv = (torch.as_tensor(np.asarray(a, np.float64)) for a in (probs, y, adv))
    lp = torch.log(p + 1e-10)
    return float((adv.reshape(-1, 1) * (-y * lp) - ent * (-p * lp)).mean())


# --------------------------------------------------------------------------------------------------------- optimiser
class KerasAdam(orc.TFAdam):
    """Keras (OptimizerV2) Adam: the tf.train.Adam update with eps 1e-7, optional per-tensor clipnorm, and `decay`:
    lr / (1 + decay * iterations) with iterations counted before the step."""

    def __init__(self, params, lr, clipnorm=None, decay=0.0, eps=1e-7):
        super().__init__(params, lr, eps=eps)
        self.base_lr, self.clipnorm, self.decay, self.iterations = lr, clipnorm, decay, 0

    def step(self, grads):
        if self.clipnorm:
            out = []
            for g in grads:
                n = float(g.double().pow(2).sum().sqrt())
                out.append(g * (self.clipnorm / n) if n > self.clipnorm else g)
            grads = out
        f = self.f
        self.lr = f(self.base_lr) / (f(1) + f(self.decay) * f(self.iterations)) if self.decay else self.base_lr
        self.iterations += 1
        super().step(grads)


def fit_batches(n, rng=np.random):
    """training_arrays.fit_loop(shuffle=True): the minibatches of one fit call."""
    order = np.arange(n)
    rng.shuffle(order)
    return [order[s:s + FIT_BATCH] for s in range(0, n, FIT_BATCH)]


class ImpalaKerasLearner:
    """ImpalaMlp / ImpalaCnn (model.fit) and IMPALA.train on torch-CPU, in the precision of xt_oracle.precision."""

    def __init__(self, arch, weights, lr=3e-4, clipnorm=None, decay=0.0, ent=0.01, gamma=0.99, batch_size=512):
        self.arch, self.names = arch, list(weights.keys())
        self.params = orc._as_param_list(weights)
        self.opt = KerasAdam(self.params, lr, clipnorm=clipnorm, decay=decay)
        self.ent, self.gamma, self.batch_size = ent, gamma, batch_size
        self.last = {}

    def weights(self):
        return OrderedDict((n, p.detach().numpy().copy()) for n, p in zip(self.names, self.params))

    def predict(self, obs):
        with torch.no_grad():
            logits, v = orc.forward(self.arch, dict(zip(self.names, self.params)), obs)
        return torch.softmax(logits, -1).numpy(), v.numpy()

    def fit(self, obs, adv, y, tv, rng=np.random):
        """model.fit(x=[obs, adv], y=[y, tv], batch_size=128): returns the epoch loss."""
        n, total = len(obs), 0.0
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, orc._PREC["np"]))   # noqa: E731
        for mb in fit_batches(n, rng):
            logits, v = orc.forward(self.arch, dict(zip(self.names, self.params)), obs[mb])
            rl = row_losses(logits, v, t(y[mb]), t(adv[mb]), t(tv[mb]), self.ent)
            grads = torch.autograd.grad(rl.mean(), self.params)
            self.opt.step(grads)
            total += float(rl.detach().sum())
        return total / n

    def train(self, trajs, rng=np.random):
        """IMPALA.train over trajectories dict(cur_state [L+1, ...], real_action [L, A], action [L, A], reward [L],
        done [L]); returns the mean slice loss."""
        L = len(trajs[0]["reward"])
        states = np.concatenate([tr["cur_state"] for tr in trajs])
        probs, values = self.predict(states)
        n = len(trajs)
        stack = lambda k: np.stack([np.asarray(tr[k]) for tr in trajs])   # noqa: E731
        pg, tv = vtrace(probs.reshape(n, L + 1, -1), values.reshape(n, L + 1), stack("action"), stack("real_action"),
                        stack("reward"), stack("done"), self.gamma)
        self.last = dict(pg_adv=pg, tv=tv)
        obs = np.concatenate([tr["cur_state"][:-1] for tr in trajs])
        amat = stack("real_action").reshape(n * L, -1)
        losses = [self.fit(obs[s:s + self.batch_size], pg[s:s + self.batch_size], amat[s:s + self.batch_size],
                           tv[s:s + self.batch_size], rng) for s in range(0, n * L, self.batch_size)]
        return float(np.mean(losses)), losses
