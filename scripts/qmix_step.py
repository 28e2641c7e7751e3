"""Time QMixModel's device training step and its one-step infer_actions on the GPU.

Sizes are qmix.yaml's (batch 32, rnn 64, mixing embed 32, hypernet embed 64); the map's sizes are arguments.  The
2s_vs_1sc defaults (2 agents, 7 actions, episode limit 300, obs 26 with the last action and agent id appended, state 27)
come from SMAC, which is not in this tree: they are unverified.  Prints one JSON line with the card's name and power
limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-agents", type=int, default=2)
    ap.add_argument("--n-actions", type=int, default=7)
    ap.add_argument("--episode-limit", type=int, default=300)
    ap.add_argument("--obs", type=int, default=26)
    ap.add_argument("--state", type=int, default=27)
    ap.add_argument("--short", type=int, default=60, help="max_ep_t of the short batch")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qmix_step.py needs a CUDA device")
    torch.cuda.set_device(0)
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import qmix_oracle as qo
    from xingtian_b200 import capi
    from xingtian_b200.model.qmix import QMixModel
    L, n = a.episode_limit, a.n_agents
    mc = dict(gamma=0.99, lr=0.0005, grad_norm_clip=10, n_agents=n, obs_shape=a.obs, rnn_hidden_dim=64, episode_limit=L,
              n_actions=a.n_actions, batch_size=32, state_shape=[a.state], mixing_embed_dim=32, hypernet_embed=64, init_seed=0)
    m = QMixModel(dict(model_config=mc, scene="train"))
    lib = capi.lib()
    res = {}
    for label, t in (("full", L + 1), ("short", a.short)):
        b = qo.synth_batch(0, 32, L, n, a.n_actions, a.obs, a.state, max_ep_t=t)
        m.train(*qo.model_args(b))
        buf = m._train_buffers()
        for _ in range(a.warmup):
            m.train_device(buf)
        torch.cuda.synchronize()
        l0 = lib.xtb_launch_count()
        t0 = time.perf_counter()
        for _ in range(a.rounds):
            m.train_device(buf)
        torch.cuda.synchronize()
        res[label + "_train_ms"] = (time.perf_counter() - t0) * 1e3 / a.rounds
        res["launches_per_step"] = (lib.xtb_launch_count() - l0) // a.rounds
    x = np.random.default_rng(0).normal(size=(1, 1, n, a.obs)).astype(np.float32)
    for _ in range(a.warmup):
        m.infer_actions(x)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.rounds * 10):
        m.infer_actions(x)
    torch.cuda.synchronize()
    res["infer_actions_ms"] = (time.perf_counter() - t0) * 1e3 / (a.rounds * 10)
    name, power = card()
    res.update(gpu=name, power_limit=power, n_agents=n, n_actions=a.n_actions, episode_limit=L, short_max_ep_t=a.short)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
