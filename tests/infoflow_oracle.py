"""Float64 restatement of the InfoFlow recommender DQN (xt/model/dqn/dqn_rec_model.py, dqn_infoflw_alg.py): the frozen
embedding, Keras's GRU v1 with hard_sigmoid gates, the dense head, mse, Keras Adam (oracle.xt_oracle.KerasAdam) and the
TD target over ragged candidates.  The arithmetic type follows oracle.xt_oracle.precision: "f64" is the yardstick, "f32"
the size of fp32 rounding.  Weights are {TF variable name: array}."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import xt_oracle as orc

HIST = 5
TRAINABLE = ["gru/kernel", "gru/recurrent_kernel", "gru/bias", "gru_1/kernel", "gru_1/recurrent_kernel", "gru_1/bias",
             "dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias", "q_value/kernel", "q_value/bias"]
ACTS = {"linear": lambda x: x, None: lambda x: x, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}


def _t(x):
    return torch.as_tensor(np.asarray(x), dtype=orc._PREC["t"])


def hard_sigmoid(x):
    return torch.clamp(0.2 * x + 0.5, 0.0, 1.0)


def gru_v1(x, w, scope, pre=None):
    """tf.keras.layers.GRU (TF 1.15, reset_after=False, zero initial state) over x [N, T, U] -> last output [N, U].
    pre (a list) collects the gate pre-activations [z | r] of every step."""
    k, rk, b = w[scope + "/kernel"], w[scope + "/recurrent_kernel"], w[scope + "/bias"]
    U = rk.shape[0]
    h = torch.zeros(x.shape[0], U, dtype=x.dtype)
    for t in range(x.shape[1]):
        xm = x[:, t] @ k + b
        zr = xm[:, :2 * U] + h @ rk[:, :2 * U]
        if pre is not None:
            pre.append(zr.detach())
        z, r = hard_sigmoid(zr[:, :U]), hard_sigmoid(zr[:, U:])
        hh = torch.tanh(xm[:, 2 * U:] + (r * h) @ rk[:, 2 * U:])
        h = z * h + (1 - z) * hh
    return h


def q_values(w, table, user, click, noclick, item, last_act, pre=None):
    """The Q value [N] of N rows of int32 ids (the tiled dict form)."""
    tb = _t(table)
    emb = lambda ids: tb[torch.as_tensor(np.asarray(ids, np.int64))]
    N = len(user)
    E = tb.shape[1]
    hc = gru_v1(emb(click).reshape(N, HIST, -1), w, "gru", pre)
    hn = gru_v1(emb(noclick).reshape(N, HIST, -1), w, "gru_1", pre)
    x = torch.cat([emb(user).reshape(N, -1), hc, hn, emb(item).reshape(N, -1)], -1)
    x = torch.relu(x @ w["dense/kernel"] + w["dense/bias"])
    x = torch.relu(x @ w["dense_1/kernel"] + w["dense_1/bias"])
    return ACTS[last_act](x @ w["q_value/kernel"] + w["q_value/bias"])[:, 0]


def td_targets(q, cand_off, reward, done, gamma):
    """dqn_infoflw_alg.py:143-153 on the Q values of the candidate rows: reward if done, else the max over the
    transition's candidates (NaN if one is NaN, as np.argmax) times gamma plus reward, in float64."""
    q = np.asarray(q)
    out = []
    for b in range(len(reward)):
        if done[b]:
            out.append(reward[b])
        else:
            seg = q[cand_off[b]:cand_off[b + 1]]
            out.append(float(np.float64(seg[np.argmax(seg)])) * gamma + reward[b])
    return np.array(out, np.float64)


class InfoflowLearner(object):
    """DqnInfoFlowModel + DQNInfoFlowAlg's step: targets from the current weights, one Keras Adam step on mse."""

    def __init__(self, weights, table, last_act, gamma, lr=0.001):
        self.w = OrderedDict((k, _t(weights[k]).clone().requires_grad_(True)) for k in TRAINABLE)
        self.table, self.last_act, self.gamma = table, last_act, gamma
        self.opt = orc.KerasAdam(list(self.w.values()), lr)

    def predict(self, user, click, noclick, item, pre=None):
        with torch.no_grad():
            return q_values(self.w, self.table, user, click, noclick, item, self.last_act, pre).numpy()

    def targets(self, b, pre=None):
        n = np.diff(b["cand_off"])
        rep = lambda a: np.repeat(a, n, axis=0)
        q = self.predict(rep(b["next_user"]), rep(b["next_click"]), rep(b["next_noclick"]), b["cand_item"], pre)
        return q, td_targets(q, b["cand_off"], b["reward"], b["done"], self.gamma).astype(np.float32)

    def step(self, b, label=None, pre=None):
        """One step; label None: the targets of the batch.  -> (loss before the update, targets)."""
        t = self.targets(b, pre)[1] if label is None else np.asarray(label, np.float32)
        y = q_values(self.w, self.table, b["user"], b["click"], b["noclick"], b["item"], self.last_act, pre)
        loss = torch.mean((y - _t(t)) ** 2)
        grads = torch.autograd.grad(loss, list(self.w.values()))
        self.opt.step(grads)
        return float(loss.detach()), t

    def weights(self):
        return OrderedDict((k, v.detach().numpy().astype(np.float64)) for k, v in self.w.items())

    def slots(self):
        return [m.numpy().astype(np.float64) for m in self.opt.m], [v.numpy().astype(np.float64) for v in self.opt.v]
