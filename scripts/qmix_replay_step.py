"""Time QMixAlg.train() and SCCAlg.train() with the host episode replay (ReplayBuffer) against the device replay
(alg_config DEVICE_REPLAY), at two map shapes, batch 32 and buffer_size 5000:

  2s_vs_1sc  2 agents, 7 actions, obs 17, state 27, episode limit 300 (QMIX at qmix.yaml's widths, SCC at scc.yaml's)
  2s3z       5 agents, 11 actions, obs 80, state 120, episode limit 120 (SCC with the agent groups [2, 3]; QMIX too)

The map sizes come from SMAC, which is not in this tree: they are unverified.  Both learners of a case share init_seed
and hold the same 64 stored episodes of random lengths (train() does not depend on how many are stored); each call
trains on the batch the last prepare_data drew.  host: the Python gather, build_inputs per step, the mask, nine staged
uploads and the model's graph; device: one staged upload of the ids, one graph (gather and step), one download.  Host
wall clock around each call up to a device synchronise; per round the two paths alternate, after a warm-up round.
Prints the card name and power limit and one JSON line of per-round medians in ms.

usage: python scripts/qmix_replay_step.py [--calls 10] [--rounds 3]"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.dueling_step import card  # noqa: E402

SHAPES = {"2s_vs_1sc": dict(n=2, A=7, obs=17, state=27, L=300, groups="2s_vs_1sc"),
          "2s3z": dict(n=5, A=11, obs=80, state=120, L=120, groups="2s3z")}


def learner(kind, s, device_replay):
    from xingtian_b200.algorithm.qmix import QMixAlg
    from xingtian_b200.algorithm.scc import SCCAlg
    env_attr = dict(n_agents=s["n"], n_actions=s["A"], state_shape=s["state"], obs_shape=s["obs"], episode_limit=s["L"])
    alg_config = dict(batch_size=32, buffer_size=5000, epsilon_anneal_time=50000, epsilon_finish=0.05, epsilon_start=1.0,
                      obs_agent_id=True, obs_last_action=True, target_update_interval=200, env_attr=env_attr,
                      instance_num=1, agent_num=1, DEVICE_REPLAY=device_replay)
    mc = dict(gamma=0.99, n_agents=s["n"], rnn_hidden_dim=64, episode_limit=s["L"], n_actions=s["A"], batch_size=32,
              state_shape=[s["state"]], use_double_q=True, init_seed=0)
    if kind == "qmix":
        mc.update(lr=0.0005, grad_norm_clip=10, mixing_embed_dim=32, hypernet_embed=64)
        return QMixAlg({"actor": {"model_name": "QMixModel", "model_config": mc}}, alg_config)
    mc.update(mixer_grad_norm_clip=5, actor_grad_norm_clip=5, a_lr=0.0005, c_lr=0.0005, dense_unit_number=128,
              enable_critic_multi_channel=True, channel_merge="concat", mc_sample_times=3, map_name=s["groups"])
    return SCCAlg({"actor": {"model_name": "SCCModel", "model_config": mc}}, alg_config)


def episode(rng, s):
    T, n, A = s["L"] + 1, s["n"], s["A"]
    m = int(rng.integers(T // 4, T + 1))
    d = dict(state=np.zeros((T, s["state"]), np.float32), obs=np.zeros((T, n, s["obs"]), np.float32),
             actions=np.zeros((T, n, 1), np.int64), avail_actions=np.zeros((T, n, A), np.int32), reward=np.zeros((T, 1), np.float32),
             terminated=np.zeros((T, 1), np.uint8), filled=np.zeros((T, 1), np.int64))
    d["state"][:m] = rng.normal(size=(m, s["state"]))
    d["obs"][:m] = rng.normal(size=(m, n, s["obs"]))
    d["avail_actions"][:m] = rng.random((m, n, A)) < 0.7
    d["avail_actions"][:m, :, 0] = 1
    d["actions"][:m, :, 0] = rng.integers(0, A, (m, n))
    d["reward"][:m, 0] = rng.normal(size=m)
    d["terminated"][m - 1] = 1
    d["filled"][:m] = 1
    return d


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    info = card()
    print(info)
    out = {}
    for shape, s in SHAPES.items():
        for kind in ("qmix", "scc"):
            algs = {"host": learner(kind, s, False), "device": learner(kind, s, True)}
            rng = np.random.default_rng(0)
            for i in range(64):
                d = episode(rng, s)
                for a in algs.values():
                    np.random.seed(i)
                    a.prepare_data({k: v.copy() for k, v in d.items()})
            res = {k: [] for k in algs}
            for r in range(args.rounds + 1):      # round 0 warms up (each path captures its graph there)
                for k, a in algs.items():
                    random.seed(r)
                    t = [wall(lambda: a.train(episode_num=1 + r * args.calls + c)) for c in range(args.calls)]
                    if r:
                        res[k].append(round(float(np.median(t)), 3))
            out["%s_%s_train_ms" % (kind, shape)] = res
            del algs
            torch.cuda.empty_cache()
    out.update(card=info, calls=args.calls, rounds=args.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
