"""Time the Muzero learner with the host replay (PrioritizedBuffer) against the device replay (alg_config DEVICE_REPLAY),
MuzeroCnn at muzero_breakout.yaml shapes (84x84x4 uint8, A = 4, K = 5):

  train_B<B>    one Muzero.train() call at B = 1024 and B = 256 over BUFFER_SIZE = B + 64 stored trajectories of 50 steps:
                host: the Python draw, gather, staged upload, model step and Python priority updates; device: 2B host
                uniforms, one staged upload, one graph replay (draw, gather, model step, updates), one download.
  prepare_L200  one Muzero.prepare_data() of a 200-step trajectory: host: value inference and the Python position tree;
                device: one staged upload, value inference from the pool rows and the tree built on the device.

Host wall clock around each call up to a device synchronise (both train() paths end in a download); per round the two
paths alternate, after warm-up calls.  The stored trajectories share one frame array on the host (the device pool holds
a copy per trajectory, and is sized so that nothing is evicted).  Prints the card name and power limit and one JSON line.

usage: python scripts/muzero_replay_step.py [--calls 10] [--rounds 3]"""
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

CFG = {"reward_min": 0, "reward_max": 50, "value_min": 0, "value_max": 500, "obs_type": "uint8", "init_seed": 0}


def learners(B, size):
    import xingtian_b200 as xb
    info = {"actor": {"model_name": "MuzeroCnn", "state_dim": [84, 84, 4], "action_dim": 4, "model_config": dict(CFG, max_batch=B)}}
    cfg = {"instance_num": 1, "agent_num": 1, "BATCH_SIZE": B, "BUFFER_SIZE": size, "UNROLL_STEP": 5}
    return {"host": xb.alg_builder("Muzero", info, cfg),
            "device": xb.alg_builder("Muzero", info, dict(cfg, DEVICE_REPLAY=True, DEVICE_REPLAY_STEPS=size * 200 + 4096))}


def trajectory(rng, frames, L):
    return dict(cur_state=frames[:L], action=rng.integers(0, 4, L), reward=rng.uniform(0, 5, L).round(1), done=np.zeros(L, bool),
                child_visits=rng.dirichlet(np.ones(4), L), target_value=rng.uniform(0, 400, L))


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
    rng = np.random.default_rng(0)
    frames = rng.integers(0, 256, (200, 84, 84, 4), dtype=np.uint8)
    out = {}
    for B in (1024, 256):
        algs = learners(B, B + 64)
        for _ in range(B + 64):
            tr = trajectory(rng, frames, 50)
            for a in algs.values():
                a.prepare_data(dict(tr))
        res = {k: [] for k in algs}
        for r in range(args.rounds + 1):           # round 0 warms up (the device path captures its graph there)
            for k, a in algs.items():
                random.seed(r)
                t = [wall(a.train) for _ in range(args.calls)]
                if r:
                    res[k].append(round(float(np.median(t)), 3))
        out["train_B%d_ms" % B] = res
        if B == 256:
            res = {k: [] for k in algs}
            for r in range(args.rounds + 1):
                for k, a in algs.items():
                    t = [wall(lambda: a.prepare_data(trajectory(rng, frames, 200))) for _ in range(args.calls)]
                    if r:
                        res[k].append(round(float(np.median(t)), 3))
            out["prepare_L200_ms"] = res
        del algs
        torch.cuda.empty_cache()
    out.update(info if isinstance(info, dict) else {"card": info})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
