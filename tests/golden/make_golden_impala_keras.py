#!/usr/bin/env python
"""Generate impala_keras.npz by EXECUTING the reference's own IMPALA learner code:

  * IMPALA.prepare_data / train / _train_proc (xt/algorithm/impala/impala.py:62-189), loaded with make_golden's stub
    modules; actor.predict is a fixed table of target probabilities / values indexed by state id and actor.train
    records the slices it is given (state ids, pg_adv, action matrix, target value).  Cases with dones, L = 1, 7, 33,
    ragged last slices and A = 2, 4, 18.
  * the `impala_loss` closures of impala_mlp.py and impala_cnn.py, run over a numpy stand-in for the two Keras backend
    ops they call (K.log, K.mean: eager float32).

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_impala_keras.py
It writes impala_keras.npz alone; the fixtures of make_golden.py are untouched."""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402


class KShim(object):
    @staticmethod
    def log(x): return np.log(np.asarray(x, np.float32)).astype(np.float32)

    @staticmethod
    def mean(x, axis=None): return np.mean(np.asarray(x, np.float32), axis=axis, dtype=np.float32)


def reference_impala():
    class Algorithm(object):
        pass
    mg.install_stubs()
    sys.modules["xt.algorithm"].Algorithm = Algorithm
    mg._load("xt.algorithm.impala.default_config", "xt/algorithm/impala/default_config.py")
    mg._mod("xt.model.tf_compat", loss_to_val=lambda x: x)
    mg._mod("xt.algorithm.alg_utils", DivideDistPolicy=object, FIFODistPolicy=object, EqualDistPolicy=object)
    return mg._load("xt.algorithm.impala.impala", "xt/algorithm/impala/impala.py")


def loss_closure(relpath):
    path = os.path.join(mg.REF, relpath)
    tree = ast.parse(open(path).read(), path)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "impala_loss"]
    assert len(keep) == 1
    ns = {"K": KShim, "ENTROPY_LOSS": 0.01}
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
    return ns["impala_loss"]


def softmax(x):
    e = np.exp(x - x.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


def golden_train_proc(ref, out):
    rng = np.random.default_rng(31)
    for case, (n_traj, L, A, batch, pdone) in enumerate([(3, 33, 4, 40, 0.1), (2, 1, 2, 512, 0.5), (4, 7, 18, 10, 0.2),
                                                         (2, 200, 2, 160, 0.02)]):
        ref.BATCH_SIZE = batch
        alg = object.__new__(ref.IMPALA)
        alg.episode_len = L
        alg._init_train_list()
        n_state = n_traj * (L + 1)
        probs = softmax(rng.standard_normal((n_state, A)).astype(np.float32) * 2)
        values = rng.standard_normal((n_state, 1)).astype(np.float32)
        slices = []

        class Actor(object):
            def predict(self, x):
                ids = np.asarray(x[0]).astype(np.int64).reshape(-1)
                return [probs[ids].copy(), values[ids].copy()]

            def train(self, state, label):
                slices.append((np.asarray(state[0]).astype(np.int64).reshape(-1), np.asarray(state[1]).reshape(-1).copy(),
                               np.asarray(label[0]).copy(), np.asarray(label[1]).reshape(-1).copy()))
                return float(len(slices))
        alg.actor = Actor()
        behav, amat, reward, done = [], [], [], []
        for t in range(n_traj):
            acts = rng.integers(0, A, L)
            tr = dict(cur_state=np.arange(t * (L + 1), (t + 1) * (L + 1), dtype=np.float32),
                      real_action=np.eye(A)[acts], action=softmax(rng.standard_normal((L, A)).astype(np.float32)),
                      reward=[float(x) for x in rng.choice([-1.0, 0.0, 1.0, 0.5], size=L)],
                      done=[bool(x) for x in (rng.random(L) < pdone)])
            behav.append(tr["action"]); amat.append(tr["real_action"]); reward.append(tr["reward"]); done.append(tr["done"])
            alg.prepare_data(tr)
        mean_loss = alg.train()
        pre = "c%d_" % case
        out.update({pre + "cfg": np.asarray([n_traj, L, A, batch]), pre + "probs": probs, pre + "values": values[:, 0],
                    pre + "behav": np.concatenate(behav), pre + "amat": np.concatenate(amat),
                    pre + "reward": np.asarray(reward, np.float64).reshape(-1), pre + "done": np.asarray(done).reshape(-1),
                    pre + "slice_sizes": np.asarray([len(s[0]) for s in slices]),
                    pre + "state_ids": np.concatenate([s[0] for s in slices]), pre + "pg_adv": np.concatenate([s[1] for s in slices]),
                    pre + "slice_amat": np.concatenate([s[2] for s in slices]), pre + "tv": np.concatenate([s[3] for s in slices]),
                    pre + "mean_loss": np.asarray(mean_loss)})


def golden_loss(out):
    rng = np.random.default_rng(32)
    mlp, cnn = loss_closure("xt/model/impala/impala_mlp.py"), loss_closure("xt/model/impala/impala_cnn.py")
    for case, (B, A, scale) in enumerate([(5, 2, 1.0), (128, 4, 3.0), (44, 18, 8.0)]):
        probs = softmax((rng.standard_normal((B, A)) * scale).astype(np.float32))
        y = np.eye(A, dtype=np.float32)[rng.integers(0, A, B)]
        adv = rng.standard_normal((B, 1)).astype(np.float32)
        pre = "loss%d_" % case
        out.update({pre + "probs": probs, pre + "y": y, pre + "adv": adv,
                    pre + "mlp": np.asarray(mlp(adv)(y, probs), np.float32), pre + "cnn": np.asarray(cnn(adv)(y, probs), np.float32)})


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        sys.exit("needs /root/reference")
    out = {}
    golden_train_proc(reference_impala(), out)
    golden_loss(out)
    np.savez(os.path.join(HERE, "impala_keras.npz"), **out)
    print("impala_keras.npz", len(out), "arrays")
