"""Time the MuZero learner on the device (xtb_muzero_*), MuzeroCnn at muzero_breakout.yaml shapes (84x84x4 uint8, A = 4,
value support 23, reward support 8, K = 5):

  train      one graph-replayed xtb_muzero_train call (with the post-update values) at B = 1024 and B = 256;
  initial    xtb_muzero_initial_inference at B = 50 (the YAML's env_num);
  recurrent  xtb_muzero_recurrent_inference at B = 50;
  gather     the learner's host side of one training call at B = 1024: the proportional sample of trajectories and
             positions, the gather of frames / actions / targets and their staged upload (xtb_copy_h2d_staged), timed on
             the host up to a stream synchronise, without the model step.

Device times: per round, warm-up replays, then CUDA events around `--replays` back-to-back calls (mean per call).  Launches
per call from xtb_launch_count around one eager call.  Prints the card name and power limit and one JSON line per item.

usage: python scripts/muzero_step.py [--replays 20] [--rounds 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.dueling_step import card  # noqa: E402

CFG = {"reward_min": 0, "reward_max": 50, "value_min": 0, "value_max": 500, "obs_type": "uint8", "init_seed": 0}


def timed(fn, replays):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / replays


def launches(fn):
    from xingtian_b200 import capi
    torch.cuda.synchronize()
    n0 = capi.lib().xtb_launch_count()
    fn()
    torch.cuda.synchronize()
    return capi.lib().xtb_launch_count() - n0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import xingtian_b200 as xb
    torch.cuda.set_device(0)
    print(card())
    rng = np.random.default_rng(0)
    out = {}
    for B in (1024, 256):
        models = {g: xb.model_builder({"model_name": "MuzeroCnn", "state_dim": [84, 84, 4], "action_dim": 4,
                                       "model_config": dict(CFG, max_batch=B, use_cuda_graph=g)}) for g in (True, False)}
        bufs = {}
        for g, m in models.items():
            b = m._buffers(B)
            b["obs"].copy_(torch.from_numpy(rng.integers(0, 256, (B, 84, 84, 4), dtype=np.uint8)))
            b["action"].copy_(torch.from_numpy(rng.integers(0, 4, (B, 5)).astype(np.int32)))
            b["tv"].copy_(torch.from_numpy(rng.uniform(0, 500, (B, 6)).astype(np.float32)))
            b["tr"].copy_(torch.from_numpy(rng.uniform(0, 50, (B, 6)).astype(np.float32)))
            b["tp"].copy_(torch.from_numpy(rng.dirichlet(np.ones(4), (B, 6)).astype(np.float32)))
            bufs[g] = b

        def step(g):
            m, b = models[g], bufs[g]
            return lambda: m.train_device(b["obs"], b["action"], b["tv"], b["tr"], b["tp"], B, b["loss"], b["value"])
        out["train_B%d" % B] = dict(us=[round(timed(step(True), args.replays), 1) for _ in range(args.rounds)],
                                    launches=launches(step(False)))
    m = xb.model_builder({"model_name": "MuzeroCnn", "state_dim": [84, 84, 4], "action_dim": 4,
                           "model_config": dict(CFG, max_batch=64)})
    obs = torch.from_numpy(rng.integers(0, 256, (50, 84, 84, 4), dtype=np.uint8)).cuda()
    _, _, hid = m.initial_inference_batch(obs, 50)
    hid = hid.clone()
    act = torch.from_numpy(rng.integers(0, 4, 50).astype(np.int32)).cuda()
    out["initial_B50"] = dict(us=[round(timed(lambda: m.initial_inference_batch(obs, 50), args.replays * 5), 1)
                                  for _ in range(args.rounds)])
    out["recurrent_B50"] = dict(us=[round(timed(lambda: m.recurrent_inference_batch(hid, act, 50), args.replays * 5), 1)
                                    for _ in range(args.rounds)])
    # host side of one learner call at B = 1024: sample, gather, staged upload
    alg = xb.alg_builder("Muzero", {"actor": {"model_name": "MuzeroCnn", "state_dim": [84, 84, 4], "action_dim": 4,
                                              "model_config": dict(CFG, max_batch=1024)}},
                         {"instance_num": 1, "agent_num": 1, "BATCH_SIZE": 1024, "BUFFER_SIZE": 2000, "UNROLL_STEP": 5})
    for _ in range(1100):
        L = 20
        alg.prepare_data(dict(cur_state=rng.integers(0, 256, (L, 84, 84, 4), dtype=np.uint8), action=rng.integers(0, 4, L),
                              reward=rng.uniform(0, 1, L), done=np.zeros(L, bool), root_value=np.zeros(L),
                              child_visits=rng.dirichlet(np.ones(4), L), target_value=rng.uniform(0, 50, L)))
    a = alg.actor
    b = a._buffers(1024)
    host = []
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, _, image, actions, tv, tr, tp = alg.sample_batch()
        for k, v, dt in (("obs", a._host_obs(image), np.uint8), ("action", actions, np.int32), ("tv", tv, np.float32),
                         ("tr", tr, np.float32), ("tp", tp, np.float32)):
            xb.engine.stage_h2d(b[k], v, dt)
        torch.cuda.synchronize()
        host.append(round((time.perf_counter() - t0) * 1e3, 2))
    out["gather_upload_B1024"] = dict(ms=host)
    for k, v in out.items():
        print(json.dumps(dict(item=k, **v)))


if __name__ == "__main__":
    main()
