"""Time SCCModel's device training step and its one-step infer_actions on the GPU.

Sizes are scc.yaml's (batch 32, rnn 64, dense_unit_number 128, mc_sample_times 3, concat multi-channel critic) in two
cases: scc.yaml's own map, 2s_vs_1sc (2 agents, 7 actions, episode limit 300, obs 26 with the last action and agent id
appended), and 2s3z with its agent groups [2, 3] (5 agents, 11 actions, raw obs 80, state 120, episode limit 120).  The
map sizes come from SMAC, which is not in this tree: they are unverified.  Prints one JSON line with the card's name and
power limit, the launches per step and the critic evaluations the reference makes per step (1 + n or 2 n mc
get_mixer_output calls for the credits, then the eval and target critics of the mixer step)."""
import argparse
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from qmix_step import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--short", type=int, default=60, help="max_ep_t of the short batch")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("scc_step.py needs a CUDA device")
    torch.cuda.set_device(0)
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import scc_oracle as so
    from xingtian_b200 import capi
    from xingtian_b200.model.scc import SCCModel
    lib = capi.lib()
    random.seed(0)
    res = {}
    for case, n, nA, L, raw, map_name in (("2s_vs_1sc", 2, 7, 300, 26 - 7 - 2, "2s_vs_1sc"), ("2s3z", 5, 11, 120, 80, "2s3z")):
        mc = dict(gamma=0.99, mixer_grad_norm_clip=5, actor_grad_norm_clip=5, a_lr=0.0005, c_lr=0.0005, rnn_hidden_dim=64,
                  batch_size=32, use_double_q=True, dense_unit_number=128, enable_critic_multi_channel=True, channel_merge="concat",
                  mc_sample_times=3, map_name=map_name, n_agents=n, n_actions=nA, obs_shape=raw + nA + n, episode_limit=L,
                  state_shape=[120], init_seed=0)
        m = SCCModel(dict(model_config=mc, scene="train"))
        r = {"reference_critic_evals_per_step": (2 * n * 3 if n > 2 else 1 + n) + 2}
        for label, t in (("full", L + 1), ("short", a.short)):
            b = so.synth_batch(0, 32, L, n, nA, raw, max_ep_t=t)
            m.train(*so.model_args(b))
            buf = m._train_buffers()
            for _ in range(a.warmup):
                m.train_device(buf)
            torch.cuda.synchronize()
            l0 = lib.xtb_launch_count()
            t0 = time.perf_counter()
            for _ in range(a.rounds):
                m.train_device(buf)
            torch.cuda.synchronize()
            r[label + "_train_ms"] = round((time.perf_counter() - t0) * 1e3 / a.rounds, 3)
            r["launches_per_step"] = (lib.xtb_launch_count() - l0) // a.rounds
        x = np.random.default_rng(0).normal(size=(1, 1, n, m.obs_shape)).astype(np.float32)
        for _ in range(a.warmup):
            m.infer_actions(x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.rounds * 10):
            m.infer_actions(x)
        torch.cuda.synchronize()
        r["infer_actions_ms"] = round((time.perf_counter() - t0) * 1e3 / (a.rounds * 10), 4)
        r.update(n_agents=n, n_actions=nA, episode_limit=L)
        res[case] = r
    name, power = card()
    res.update(gpu=name, power_limit=power, short_max_ep_t=a.short)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
