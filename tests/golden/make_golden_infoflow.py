#!/usr/bin/env python
"""Generate infoflow.npz by EXECUTING the reference's own DQNInfoFlowAlg (xt/algorithm/dqn/dqn_infoflw_alg.py) and its
ReplayBuffer (xt/algorithm/replay_buffer.py) over the seeded session of tests/infoflow_alg_scenario.py, with a recording
stand-in actor: its predict returns seeded Q values, its train records its arguments and shuffles np.arange(batch_size)
with the global NumPy stream as Keras's fit does, and get_weights / set_weights mark the target syncs.  The registry, the
Algorithm base (which only builds the actor) and model_builder are stubbed.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_infoflow.py
It writes infoflow.npz alone."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402
import infoflow_alg_scenario as sc  # noqa: E402

REC = sc.Recorder()


class RecordingActor(object):
    def __init__(self, model_info):
        self.model_info = model_info

    def predict(self, state):
        REC.predicts.append({k: np.asarray(v).copy() for k, v in state.items()})
        q = REC.q_values(len(state["item_input"]))
        REC.predicts[-1]["q"] = q
        return q

    def train(self, state, label, batch_size, verbose=False):
        REC.trains.append(({k: np.asarray(v).copy() for k, v in state.items()}, np.asarray(label).copy(), batch_size))
        np.random.shuffle(np.arange(len(label)))      # training_arrays.fit_loop's shuffle
        return 0.0

    def get_weights(self):
        return ["weights"]

    def set_weights(self, weights):
        REC.syncs.append(len(REC.trains))


def main():
    mg.install_stubs()
    mg._mod("xt.model", model_builder=RecordingActor)

    class Algorithm(object):
        def __init__(self, alg_name, model_info, alg_config=None, **kwargs):
            self.actor = RecordingActor(model_info)
            self.alg_name, self.model_info, self.alg_config = alg_name, model_info, alg_config

    sys.modules["xt.algorithm"].Algorithm = Algorithm
    mg._load("xt.algorithm.dqn.default_config", "xt/algorithm/dqn/default_config.py")
    mg._load("xt.algorithm.replay_buffer", "xt/algorithm/replay_buffer.py")
    alg_mod = mg._load("xt.algorithm.dqn.dqn_infoflw_alg", "xt/algorithm/dqn/dqn_infoflw_alg.py")
    model_info, alg_config = sc.configs()
    alg = alg_mod.DQNInfoFlowAlg(model_info, alg_config)
    out = sc.drive(alg, REC)
    save = dict(n_trained=np.array(out["n_trained"]), synced_after_train=np.array(out["synced_after_train"], np.int64),
                py_state=np.stack(out["py_state"]), np_key=np.stack(out["np_key"]), np_pos=np.array(out["np_pos"]))
    for i, (p, (state, label, bs)) in enumerate(zip(REC.predicts, REC.trains)):
        for k, v in p.items():
            save["t%d_next_%s" % (i, k)] = v
        for k, v in state.items():
            save["t%d_%s" % (i, k)] = v
        save["t%d_target" % i] = label
        save["t%d_batch_size" % i] = np.array(bs)
    np.savez_compressed(os.path.join(HERE, "infoflow.npz"), **save)
    print("infoflow.npz: %d train calls, syncs after trains %s" % (out["n_trained"], out["synced_after_train"]))


if __name__ == "__main__":
    main()
