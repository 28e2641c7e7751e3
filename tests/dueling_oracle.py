"""The dueling Q head on top of the oracle (oracle/xt_oracle.py), for the tests of the "dueling" layer kind.

The reference builds it in xt/model/dqn/dqn_cnn.py:53-58 and dqn_mlp.py:50-54,80-87:
    value = Dense(A, linear)(dense);  adv = Dense(1, linear)(dense)
    Q = adv + (value - reduce_mean(value, axis=1, keep_dims=True))
A layer ("name", "dueling", (value_src, adv_src), {}) owns no variables.  Every other layer goes through the oracle
unchanged, in the oracle's precision (orc.precision)."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import xt_oracle as orc


def combine(value, adv):
    """Q = adv + (value - mean over actions of value), the reference's arithmetic and names."""
    return adv + (value - value.mean(dim=1, keepdim=True))


def _split(arch):
    """arch without its dueling layers (their sources become outputs), and the dueling layers"""
    duel = [l for l in arch["layers"] if l[1] == "dueling"]
    rest = [l for l in arch["layers"] if l[1] != "dueling"]
    outs = [n for n in arch["outputs"] if n not in {d[0] for d in duel}]
    for _, _, (v, a), _ in duel:
        outs += [v, a]
    return dict(arch, layers=rest, outputs=outs), duel


def dqn_cnn_arch(state_dim=(84, 84, 4), action_dim=4, dueling=False):
    arch = orc.dqn_cnn_arch(state_dim, action_dim)
    if dueling:
        arch["layers"].append(("dense_2", "dense", "dense", dict(n=1, act=None)))
        arch["layers"].append(("dueling", "dueling", ("dense_1", "dense_2"), {}))
        arch["outputs"] = ["dueling"]
    return arch


def dqn_mlp_arch(state_dim=(4,), action_dim=2, hidden_size=128, num_layers=1, dueling=False):
    arch = orc.dqn_mlp_arch(state_dim, action_dim, hidden_size, num_layers)
    if dueling:
        hidden = "dense" if num_layers == 1 else "dense_%d" % (num_layers - 1)
        arch["layers"].append(("dense_%d" % (num_layers + 1), "dense", hidden, dict(n=1, act=None)))
        arch["layers"].append(("dueling", "dueling", ("dense_%d" % num_layers, "dense_%d" % (num_layers + 1)), {}))
        arch["outputs"] = ["dueling"]
    return arch


def tensor_shapes(arch):
    base, duel = _split(arch)
    shapes = orc.tensor_shapes(base)
    for name, _, (v, _), _ in duel:
        shapes[name] = shapes[v]
    return shapes


def param_shapes(arch):
    return orc.param_shapes(_split(arch)[0])


def init_weights(arch, seed=0):
    return orc.init_weights(_split(arch)[0], seed=seed)


def forward(arch, weights, obs, keep=False):
    base, duel = _split(arch)
    t = orc.forward(base, weights, obs, keep=True)
    for name, _, (v, a), _ in duel:
        t[name] = combine(t[v], t[a])
    if keep:
        return t
    return [t[o] for o in arch["outputs"]]


class DqnLearner(orc.DqnLearner):
    """orc.DqnLearner on an arch that may hold a dueling layer; n_step / huber extend the TD target and loss the way
    xtb_dqn_td_loss_grad does (disc per row, Huber with that delta)."""

    def predict(self, states, target=False):
        w = dict(zip(self.names, self.target if target else self.params))
        with torch.no_grad():
            return forward(self.arch, w, states)[0].numpy()

    def loss_and_grads(self, states, actions, rewards, new_states, dones, disc=None, huber=0.0):
        y_t = self.predict(states)
        tq = self.predict(new_states, target=True)
        qn = self.predict(new_states) if self.double else None
        if disc is None:
            y = orc.dqn_targets(y_t, tq, actions, rewards, dones, self.gamma, qn)
        else:
            y = np.array(y_t, copy=True)
            best = np.argmax(qn, 1) if qn is not None else np.argmax(tq, 1)
            for k in range(len(y)):
                y[k][actions[k]] = rewards[k] if dones[k] else rewards[k] + disc[k] * tq[k, best[k]]
        w = dict(zip(self.names, self.params))
        q = forward(self.arch, w, states)[0]
        diff = q - torch.from_numpy(y)
        if huber > 0:
            ad = diff.abs()
            per = torch.where(ad <= huber, 0.5 * diff * diff, huber * (ad - 0.5 * huber))
        else:
            per = diff * diff
        loss = per.mean()
        return loss, torch.autograd.grad(loss, self.params), y

    def train(self, states, actions, rewards, new_states, dones, disc=None, huber=0.0):
        loss, grads, _ = self.loss_and_grads(states, actions, rewards, new_states, dones, disc, huber)
        if self.clipnorm:
            cg = []
            for g in grads:
                n = float(g.double().pow(2).sum().sqrt())
                cg.append(g * (self.clipnorm / n) if n > self.clipnorm else g)
            grads = cg
        self.opt.step(grads)
        self.train_count += 1
        if self.train_count % self.freq == 0:
            self.target = [p.detach().clone() for p in self.params]
        return float(loss.detach())


def weights_in_order(arch, w):
    return OrderedDict((k, w[k]) for k in param_shapes(arch))
