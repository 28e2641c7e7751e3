#!/usr/bin/env python
"""Generate scc.npz by EXECUTING the reference's own SCC host code:

- an SCCAlg session (xt/algorithm/scc/scc_alg.py with the QMIX episode buffer and transforms it imports), driven through
  the seeded session of tests/qmix_alg_scenario.py with its recording stand-in actor, which records every argument of
  train, the raw observations included (keys "alg_*");
- SCCModel.train's NumPy part (xt/model/scc/scc_tf.py:535-564 with the credit methods of 657-707) on an instance made
  without __init__: get_mixer_output is a float64 critic (_build_mixer's arithmetic) whose weights are stored here, and
  train_mixer / train_policy record what they receive (keys "c<k>_*").  Cases: n_agents 2 (mask credits) and 3 and 5
  (Monte-Carlo credits from the seeded global `random`), concat, add and single-channel critics, a grouped map.  The
  state of `random` after each call is recorded.

tf, absl, the registry and the Algorithm base are stubbed as in make_golden_qmix.py.
Run in the build container only (needs the reference tree):  python tests/golden/make_golden_scc.py
It writes scc.npz alone."""
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402
import qmix_alg_scenario as sc  # noqa: E402

TRAIN_NAMES = ("trajectories", "obs", "obs_len", "avail", "actions", "cur_stats", "target_stats", "rewards", "terminated", "mask")
# (n_agents, multi-channel, channel_merge, groups, mc_sample_times)
CASES = [(2, True, "concat", [2], 1), (2, False, None, [2], 1), (3, True, "add", [3], 3), (3, False, None, [3], 2),
         (5, True, "concat", [2, 3], 3), (5, True, "add", [2, 3], 2), (5, False, None, [5], 1)]
B, L, O, A, U = 2, 4, 3, 4, 6


def critic64(w, s, n, multi, merge, groups):
    """_build_mixer (scc_tf.py:278-313) in float64 on states [B, L, n D] -> [B, L, 1]."""
    relu = lambda x: np.maximum(x, 0.0)   # noqa: E731
    mlp = lambda p, x: relu(relu(x @ w[p + "dense/kernel"] + w[p + "dense/bias"]) @ w[p + "dense_1/kernel"] + w[p + "dense_1/bias"])  # noqa: E731
    if not multi:
        return mlp("critic/", s) @ w["v/kernel"] + w["v/bias"]
    x = s.reshape(s.shape[0], s.shape[1], n, -1)
    hs, a = [], 0
    for j, g in enumerate(groups):
        for i in range(a, a + g):
            hs.append(mlp("channel_%d/" % j, x[:, :, i]))
        a += g
    h = np.concatenate(hs, 2) if merge == "concat" else sum(hs[1:], hs[0])
    return h @ w["v/kernel"] + w["v/bias"]


def critic_weights(rng, n, multi, merge, groups):
    D, w = O + A, {}
    for j, scope in enumerate(["channel_%d/" % j for j in range(len(groups))] if multi else ["critic/"]):
        width = D if multi else n * D
        for name, shape in (("dense/kernel", (width, U)), ("dense/bias", (U,)), ("dense_1/kernel", (U, U)), ("dense_1/bias", (U,))):
            w[scope + name] = rng.normal(size=shape) * 0.5
    w["v/kernel"] = rng.normal(size=(n * U if multi and merge == "concat" else U, 1))
    w["v/bias"] = rng.normal(size=(1,))
    return w


def model_cases(ref):
    out = {}
    for k, (n, multi, merge, groups, mc) in enumerate(CASES):
        rng = np.random.default_rng(300 + k)
        w = critic_weights(rng, n, multi, merge, groups)
        m = object.__new__(ref.SCCModel)
        m.n_agents, m.n_actions, m.batch_size, m.o_shape = n, A, B, O
        m.model_config = {"mc_sample_times": mc}
        m.get_mixer_output = lambda s, w=w, n=n, multi=multi, merge=merge, groups=groups: critic64(w, s, n, multi, merge, groups)
        got = {}

        def train_mixer(*args):
            got["mixer_state"], got["next_mixer_state"] = np.array(args[-2]), np.array(args[-1])
            got["same_object"] = args[-2] is args[-1]
            return np.float32(1.5)

        def train_policy(*args):
            got["target_q_val"] = np.array(args[-1])
            return np.float32(0.25)

        m.train_mixer, m.train_policy = train_mixer, train_policy
        obs = rng.normal(size=(B, L + 1, n, O)).astype(np.float32)
        actions = rng.integers(0, A, size=(B, L, n, 1)).astype(np.int64)
        actions[:, -1] = 0     # a padding step: action 0
        random.seed(1000 + k)
        loss = m.train(None, obs, None, None, actions, None, None, None, None, None)
        state = random.getstate()
        out["c%d_obs" % k], out["c%d_actions" % k] = obs, actions
        out["c%d_mixer_state" % k] = got["mixer_state"]
        out["c%d_target_q_val" % k] = got["target_q_val"]
        out["c%d_aliased" % k] = np.array(got["same_object"])
        out["c%d_loss" % k] = np.asarray(loss)
        out["c%d_random_state" % k] = np.array(state[1], np.int64)
        out["c%d_config" % k] = np.array([n, int(multi), {None: -1, "concat": 0, "add": 1}[merge], mc] + groups)
        for name, v in w.items():
            out["c%d_w_%s" % (k, name)] = v
    return out


def alg_session(alg_mod, ebn, tr):
    model_info, alg_config = sc.configs()
    alg = alg_mod.SCCAlg(model_info, alg_config)

    def new_episode_batch(a):
        pre = {"actions": ("actions_onehot", [tr.OneHotNp(out_dim=sc.N_ACTIONS)])}
        return ebn.EpisodeBatchNP(a.scheme, a.groups, 1, sc.LIMIT + 1, preprocess=pre)

    out = sc.drive(alg, new_episode_batch)
    # the scenario names QMixAlg's nine train arguments; SCCAlg passes ten
    out = {k: v for k, v in out.items() if not k.startswith("train")}
    for k, args in enumerate(alg.actor.trained):
        for name, a in zip(TRAIN_NAMES, args):
            out["train%d_%s" % (k, name)] = a
    out["alg_name"] = np.array(alg.alg_name)
    try:
        alg_mod.SCCAlg(*sc.configs()).train_ready(0)
        out["train_ready_error"] = np.array("")
    except KeyError as e:
        out["train_ready_error"] = np.array(str(e.args[0]))
    return {"alg_" + k: v for k, v in out.items()}


def main():
    if not hasattr(np, "float"):
        np.float = float
    mg.install_stubs()
    for pkg in ("xt.algorithm.qmix", "xt.algorithm.scc", "xt.model.scc"):
        mg._mod(pkg).__path__ = []
    mg._mod("xt.model.tf_compat", tf=types.SimpleNamespace(float32=np.float32))
    mg._mod("xt.model.tf_utils", TFVariables=object)

    class Algorithm(object):
        def __init__(self, alg_name, model_info, alg_config=None, **kwargs):
            self.actor = sc.RecordingActor(model_info)
            self.alg_name, self.model_info, self.alg_config = alg_name, model_info, alg_config

    sys.modules["xt.algorithm"].Algorithm = Algorithm
    mg._mod("xt.algorithm.algorithm", ZFILL_LENGTH=5)
    ebn = mg._load("xt.algorithm.qmix.episode_buffer_np", "xt/algorithm/qmix/episode_buffer_np.py")
    tr = mg._load("xt.algorithm.qmix.transforms", "xt/algorithm/qmix/transforms.py")
    alg_mod = mg._load("xt.algorithm.scc.scc_alg", "xt/algorithm/scc/scc_alg.py")
    alg_mod.print = lambda *a, **k: None
    ref = mg._load("xt.model.scc.scc_tf", "xt/model/scc/scc_tf.py")
    out = alg_session(alg_mod, ebn, tr)
    out.update(model_cases(ref))
    np.savez(os.path.join(HERE, "scc.npz"), **out)
    print("scc.npz: %d train calls, %d model cases" % (int(out["alg_n_trained"]), len(CASES)))


if __name__ == "__main__":
    main()
