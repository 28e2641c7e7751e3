#!/usr/bin/env python
"""Generate qmix.npz by EXECUTING the reference's own QMIX host code: EpisodeBatchNP / ReplayBufferNP
(xt/algorithm/qmix/episode_buffer_np.py), OneHotNp (xt/algorithm/qmix/transforms.py) and QMixAlg with its
DecayThenFlatSchedule and EpsilonGreedyActionSelector (xt/algorithm/qmix/qmix_alg.py), driven through the seeded session
of tests/qmix_alg_scenario.py with its recording stand-in actor.  tf, absl, the registry and the Algorithm base are
stubbed (the base only builds the actor and keeps alg_config); NumPy 2 has no np.float, which the reference reads, so it
is provided as Python's float (its meaning in the NumPy the reference was written for).

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_qmix.py
It writes qmix.npz alone."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402
import qmix_alg_scenario as sc  # noqa: E402


def main():
    if not hasattr(np, "float"):
        np.float = float
    mg.install_stubs()
    for pkg in ("xt.algorithm.qmix",):
        mg._mod(pkg).__path__ = []
    mg._mod("xt.model.tf_compat", tf=types.SimpleNamespace(float32=np.float32))

    class Algorithm(object):
        def __init__(self, alg_name, model_info, alg_config=None, **kwargs):
            self.actor = sc.RecordingActor(model_info)
            self.alg_name, self.model_info, self.alg_config = alg_name, model_info, alg_config

    sys.modules["xt.algorithm"].Algorithm = Algorithm
    mg._mod("xt.algorithm.algorithm", ZFILL_LENGTH=5)
    ebn = mg._load("xt.algorithm.qmix.episode_buffer_np", "xt/algorithm/qmix/episode_buffer_np.py")
    tr = mg._load("xt.algorithm.qmix.transforms", "xt/algorithm/qmix/transforms.py")
    alg_mod = mg._load("xt.algorithm.qmix.qmix_alg", "xt/algorithm/qmix/qmix_alg.py")
    alg_mod.print = lambda *a, **k: None
    model_info, alg_config = sc.configs()
    alg = alg_mod.QMixAlg(model_info, alg_config)

    def new_episode_batch(a):
        pre = {"actions": ("actions_onehot", [tr.OneHotNp(out_dim=sc.N_ACTIONS)])}
        return ebn.EpisodeBatchNP(a.scheme, a.groups, 1, sc.LIMIT + 1, preprocess=pre)

    out = sc.drive(alg, new_episode_batch)
    out["model_obs_shape"] = np.array(model_info["actor"]["model_config"]["obs_shape"])
    out["scene"] = np.array(model_info["actor"]["scene"])
    np.savez(os.path.join(HERE, "qmix.npz"), **out)
    print("qmix.npz: %d train calls, %d episode draws, syncs after trains %s" % (out["n_trained"], out["n_sampled"],
                                                                              out["synced_after_train"].tolist()))


if __name__ == "__main__":
    main()
