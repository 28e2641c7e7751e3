#!/usr/bin/env python
"""Generate muzero.npz by EXECUTING the reference's own MuZero code:

* value_compression / value_decompression (xt/model/muzero/muzero_utils.py:38-47);
* MuzeroModel.conver_value / value_transform (xt/model/muzero/muzero_model.py:200-226), with np.asscalar (removed from
  numpy) shimmed as .item();
* the Muzero learner's prepare_data / train / sample_position / make_target / calc_pri / update_pri
  (xt/algorithm/muzero/muzero.py) over the reference's PrioritizedReplayBuffer and segment trees
  (xt/algorithm/prioritized_replay_buffer_muzero.py, xt/algorithm/segment_tree.py), under random.seed, with a stand-in
  model whose value_inference is a fixed function of the observation (value = 0.01 * sum of the observation row) and
  whose train records its minibatch and returns 0.  This pins the sampled trajectories and positions, the gathered
  minibatch and every priority, including the reference's quirks: update_pri writes the trajectory weight at the batch
  position, and _sample_proportional's total excludes the last stored item.
* the int8 feed cast of obs_type int8: np.asarray(uint8 frame, dtype=np.int8) / 255 for every byte (TF 1's feed_dict
  converts with numpy; not run under TF).

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_muzero.py
It writes muzero.npz alone."""
import ast
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402


def _defs(rel, names=None, cls=None):
    path = os.path.join(mg.REF, rel)
    tree = ast.parse(open(path).read(), path)
    body = tree.body
    if cls is not None:
        body = [n for n in body if isinstance(n, ast.ClassDef) and n.name == cls][0].body
    keep = [n for n in body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and (names is None or n.name in names)]
    return ast.Module(body=keep, type_ignores=[]), path


def _exec(rel, ns, names=None, cls=None):
    mod, path = _defs(rel, names, cls)
    exec(compile(mod, path, "exec"), ns)
    return ns


class _NpShim(types.ModuleType):
    def __getattr__(self, k):
        return getattr(np, k)


def main():
    out = {}
    npx = _NpShim("numpy")
    npx.asscalar = lambda a: np.asarray(a).item()
    utils = _exec("xt/model/muzero/muzero_utils.py", {"np": np}, names=("value_compression", "value_decompression"))
    x = np.concatenate([np.linspace(-400, 400, 97), np.linspace(0, 60000, 61), [0.0, 1e-3, -1e-3]])
    out["h_x"] = x
    out["h"] = utils["value_compression"](x)
    out["h_inv"] = utils["value_decompression"](out["h"])
    model = _exec("xt/model/muzero/muzero_model.py", dict(np=npx, value_compression=utils["value_compression"],
                                                          value_decompression=utils["value_decompression"]),
                  names=("conver_value", "value_transform"), cls="MuzeroModel")
    rng = np.random.default_rng(11)
    for tag, (lo, hi) in (("breakout_v", (0, 500)), ("breakout_r", (0, 50)), ("pong_v", (-21, 21)), ("pong_r", (-2, 2)),
                          ("default_v", (0, 60000))):
        S = int(np.ceil(utils["value_compression"](hi - lo))) + 1
        # inside the range: conver_value indexes floor + 1, which runs past the support at the top of the range
        tv = rng.uniform(lo - 3, hi - 1e-3 * (hi - lo), (7, 6))
        out["cv_in_" + tag] = tv
        out["cv_" + tag] = model["conver_value"](None, tv, S, lo, hi)
        probs = rng.dirichlet(np.ones(S), 9)
        out["vt_in_" + tag] = probs
        out["vt_" + tag] = np.array([model["value_transform"](None, p, S, lo, hi) for p in probs])
    # the learner over the reference buffer
    seg = _exec("xt/algorithm/segment_tree.py", {"operator": __import__("operator")})
    prb = _exec("xt/algorithm/prioritized_replay_buffer_muzero.py", dict(seg, random=random, np=np))
    K, B, NBUF, A = 5, 6, 8, 3
    alg = _exec("xt/algorithm/muzero/muzero.py", dict(np=np, PrioritizedReplayBuffer=prb["PrioritizedReplayBuffer"], BATCH_SIZE=B),
                names=("prepare_data", "train", "sample_position", "make_target", "calc_pri", "update_pri"), cls="Muzero")
    trained = []

    class Actor(object):
        def value_inference(self, s):
            return 0.01 * np.asarray(s, np.float64).reshape(len(s), -1).sum(1)

        def train(self, state, label):
            trained.append((np.asarray(state[0]), np.asarray(state[1]), [np.asarray(v) for v in label]))
            return 0.0

    learner = types.SimpleNamespace(buff=prb["PrioritizedReplayBuffer"](NBUF, alpha=1), unroll_step=K, actor=Actor())
    for name, fn in alg.items():
        if callable(fn) and name in ("prepare_data", "train", "sample_position", "make_target", "calc_pri", "update_pri"):
            setattr(learner, name, types.MethodType(fn, learner))
    trajs = []
    for t in range(22):     # more than NBUF: the ring wraps
        L = int(rng.integers(4, 15))   # some too short to keep
        tr = dict(cur_state=rng.normal(size=(L, 4)).round(3), action=rng.integers(0, A, L), reward=rng.normal(size=L).round(3),
                  done=np.zeros(L, bool), root_value=rng.normal(size=L), child_visits=rng.dirichlet(np.ones(A), L),
                  target_value=rng.normal(size=L).round(3), traj_id=t)
        trajs.append(tr)
        out["traj%d_len" % t] = np.array(L)
        for k in ("cur_state", "action", "reward", "child_visits", "target_value"):
            out["traj%d_%s" % (t, k)] = np.asarray(tr[k])
    random.seed(1234)
    for t, tr in enumerate(trajs):
        learner.prepare_data(dict(tr))
        if t in (3, 12, 21):     # at 3 the buffer holds fewer than B trajectories: train returns 0 and draws nothing
            for _ in range(3):
                learner.train()
    out["n_train_steps"] = np.array(len(trained))
    for s, (img, act, (tv, tr_, tp)) in enumerate(trained):
        out["step%d_image" % s], out["step%d_action" % s] = img, act
        out["step%d_tv" % s], out["step%d_tr" % s], out["step%d_tp" % s] = tv, tr_, tp
    buf = learner.buff
    out["buf_len"] = np.array(len(buf._storage))
    out["buf_ids"] = np.array([d["traj_id"] for d in buf._storage])
    out["buf_pri"] = np.array([buf._it_sum[i] for i in range(len(buf._storage))])
    out["buf_pos_pri"] = np.concatenate([[d["pos_buff"]._it_sum[i] for i in range(len(d["pos_buff"]._storage))]
                                         for d in buf._storage])
    # the int8 feed cast
    out["int8_cast"] = np.asarray(np.arange(256, dtype=np.uint8), dtype=np.int8).astype(np.float64) / 255.0
    np.savez(os.path.join(HERE, "muzero.npz"), **out)


if __name__ == "__main__":
    main()
