"""CPU oracle for IMPALA with the Keras learner (xt/algorithm/impala/impala.py, xt/model/impala/impala_mlp.py and
impala_cnn.py), on top of oracle/xt_oracle.py.  TEST INFRASTRUCTURE ONLY.

Pinned by tests/golden/impala_keras.npz (the reference's own _train_proc / train slicing and impala_loss closures,
executed by tests/golden/make_golden_impala_keras.py): the V-trace variant, the slices, the loss value.  Restated from
documented TF-1.15 behaviour and unpinned, like tf.train.AdamOptimizer and KerasAdam in xt_oracle:
  * training_arrays.fit_loop: one np.random.shuffle(np.arange(n)) per fit call, consecutive batches of 128, the last
    one ragged;
  * the epoch loss fit reports: per-batch losses weighted by batch size, i.e. sum over rows of the row loss / n."""
import numpy as np
import torch

from oracle import xt_oracle as orc

FIT_BATCH = 128


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


def fit_batches(n, rng=np.random):
    """training_arrays.fit_loop(shuffle=True): the minibatches of one fit call."""
    order = np.arange(n)
    rng.shuffle(order)
    return [order[s:s + FIT_BATCH] for s in range(0, n, FIT_BATCH)]


class ImpalaKerasLearner(orc.Learner):
    """ImpalaMlp / ImpalaCnn (model.fit) and IMPALA.train on torch-CPU, in the precision of xt_oracle.precision; the
    archs are xt_oracle.impala_mlp_arch / impala_keras_cnn_arch."""

    def __init__(self, arch, weights, lr=3e-4, clipnorm=None, decay=0.0, ent=0.01, gamma=0.99, batch_size=512):
        super().__init__(arch, weights)
        self.opt = orc.KerasAdam(self.params, lr, clipnorm=clipnorm, decay=decay)
        self.ent, self.gamma, self.batch_size = ent, gamma, batch_size
        self.last = {}

    def predict(self, obs):
        with torch.no_grad():
            logits, v = orc.forward(self.arch, self.named(), obs)
        return torch.softmax(logits, -1).numpy(), v.numpy()

    def fit(self, obs, adv, y, tv, rng=np.random):
        """model.fit(x=[obs, adv], y=[y, tv], batch_size=128): returns the epoch loss."""
        n, total = len(obs), 0.0
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, orc._PREC["np"]))   # noqa: E731
        for mb in fit_batches(n, rng):
            logits, v = orc.forward(self.arch, self.named(), obs[mb])
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
