"""Time one MuZero tree search step of N = 50 environments with S = 50 simulations (the env_num and NUM_SIMULATIONS of
muzero_breakout.yaml and muzero_pong.yaml), MuzeroCnn at both configs' shapes (84x84x4; breakout A = 4 uint8, pong A = 6
int8), three ways, rounds alternated:

  device      xtb_muzero_search: the initial inference, S x (select, recurrent inference, expand + backup) and the result
              kernel as one graph-replayed call on device observations (results stay on the device);
  host_tree   the same search with the trees on the host (tests/mcts_oracle.py, float64 lock step) and one batched
              recurrent_inference_batch per simulation, each followed by its download;
  reference   the reference's shape: per environment one initial_inference and S recurrent_inference batch-1 host calls
              (MuzeroModel.initial_inference / recurrent_inference), with the tree on the host.  Timed over the first
              --ref-envs environments and scaled to N (stated in the output).

Times are host wall clock up to a stream synchronise, per search of all N environments.  Launches per search from
xtb_launch_count around one call.  Prints the card name and power limit and one JSON line per item.

usage: python scripts/muzero_search.py [--rounds 3] [--reps 5] [--ref-envs 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from scripts.dueling_step import card  # noqa: E402
import mcts_oracle as mo  # noqa: E402

CONFIGS = {
    "breakout": (4, {"reward_min": 0, "reward_max": 50, "value_min": 0, "value_max": 500, "obs_type": "uint8"}),
    "pong": (6, {"reward_min": -2, "reward_max": 2, "value_min": -21, "value_max": 21, "obs_type": "int8"}),
}
N, S = 50, 50


def wall(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e6 / reps


def launches(fn):
    from xingtian_b200 import capi
    torch.cuda.synchronize()
    n0 = capi.lib().xtb_launch_count()
    fn()
    torch.cuda.synchronize()
    return capi.lib().xtb_launch_count() - n0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-envs", type=int, default=5)
    args = ap.parse_args()
    import xingtian_b200 as xb
    torch.cuda.set_device(0)
    print(card())
    for name, (A, cfg) in CONFIGS.items():
        m = xb.model_builder({"model_name": "MuzeroCnn", "state_dim": [84, 84, 4], "action_dim": A,
                              "model_config": dict(cfg, init_seed=0, max_batch=64)})
        rng = np.random.default_rng(0)
        obs = rng.integers(0, 256, (N, 84, 84, 4), dtype=np.uint8)
        noise = rng.dirichlet([0.25] * A, N)
        obs_dev = m._buffers(N)["obs"]
        obs_dev.copy_(torch.from_numpy(m._host_obs(obs)))
        noise_dev = torch.from_numpy(noise).cuda()

        def device():
            m.search_device(obs_dev, N, S, noise_dev)

        def host_tree():
            def initial(_):
                _, policy, hidden = m.initial_inference_batch(obs_dev, N)
                return policy.cpu().numpy(), list(hidden.clone())

            def recurrent(rows, actions):
                value, reward, policy, hid = m.recurrent_inference_batch(torch.stack(rows), torch.tensor(actions, dtype=torch.int32,
                                                                                                       device=m.device), N)
                return value.cpu().numpy(), reward.cpu().numpy(), policy.cpu().numpy(), list(hid.clone())
            return mo.search(initial, recurrent, obs, S, noise)

        k = args.ref_envs

        def reference():
            def initial(o):
                out = [m.initial_inference(x[None]) for x in o]
                return np.stack([r.policy for r in out]), [r.hidden_state for r in out]

            def recurrent(hidden, actions):
                out = [m.recurrent_inference(h, a) for h, a in zip(hidden, actions)]
                return [r.value for r in out], [r.reward for r in out], np.stack([r.policy for r in out]), [r.hidden_state for r in out]
            for e in range(k):
                mo.search(initial, recurrent, obs[e:e + 1], S, noise[e:e + 1])

        res = {"device": [], "host_tree": [], "reference": []}
        device(); host_tree(); reference()   # warm-up: graph captures, buffers
        for _ in range(args.rounds):
            res["device"].append(wall(device, args.reps * 10))
            res["host_tree"].append(wall(host_tree, args.reps))
            res["reference"].append(wall(reference, 1) * N / k)
        launch = {"device": launches(device), "host_tree": launches(host_tree), "reference": launches(reference) * N // k}
        # the device search and the host-tree search reach the same visit counts
        counts, _ = m.search_device(obs_dev, N, S, noise_dev)
        hc, _, margin = host_tree()
        for item, us in res.items():
            line = dict(item="%s_%s" % (name, item), A=A, N=N, S=S, us_per_search=[round(u, 1) for u in us],
                        launches_per_search=launch[item])
            if item == "reference":
                line["note"] = "first %d environments timed, scaled to %d" % (k, N)
            if item == "device":
                line["counts_equal_host_tree"] = bool(np.array_equal(counts.cpu().numpy(), hc))
                line["min_ucb_margin"] = margin
            print(json.dumps(line))


if __name__ == "__main__":
    main()
