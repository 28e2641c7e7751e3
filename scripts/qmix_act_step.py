"""Time one QMixModel.act call over N environments against N one-environment steps of the host path
(QMixModel.infer_actions, then EpsilonGreedyActionSelector.select_action on the host), for N in 1, 8, 64, 256, 1024.

Widths are qmix.yaml's (rnn 64) in the explore scene, inputs with the last action and the agent id appended.  Maps:
2s_vs_1sc at the sizes scripts/qmix_step.py uses (2 agents, 7 actions, obs 26 with both one-hots, so 17 raw) and a larger
one (8 agents, 14 actions, 80 raw obs); both come from SMAC, which is not in this tree, so they are unverified.
act_ms: host arrays in, host actions out (uploads, one graph, one download); act_device_ms: the same on device tensors;
host_ms: the N host-path steps, run one after another.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from qmix_step import card  # noqa: E402

MAPS = {"2s_vs_1sc": (2, 7, 17), "8a_14act_obs80": (8, 14, 80)}


def timed(fn, rounds):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", default="1,8,64,256,1024")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--host-rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qmix_act_step.py needs a CUDA device")
    torch.cuda.set_device(0)
    from xingtian_b200.algorithm.qmix import EpsilonGreedyActionSelector
    from xingtian_b200.model.qmix import QMixModel
    envs = [int(x) for x in a.envs.split(",")]
    sel = EpsilonGreedyActionSelector(dict(epsilon_start=1.0, epsilon_finish=0.05, epsilon_anneal_time=50000))
    res = {}
    for name, (n, A, o) in MAPS.items():
        mc = dict(n_agents=n, obs_shape=o + A + n, rnn_hidden_dim=64, episode_limit=300, n_actions=A, batch_size=32, state_shape=[27],
                  mixing_embed_dim=32, hypernet_embed=64, init_seed=0, act_envs=max(envs), obs_last_action=True, obs_agent_id=True)
        m = QMixModel(dict(model_config=mc, scene="explore"))
        rng = np.random.default_rng(0)
        rows = []
        for N in envs:
            obs = rng.normal(size=(N, n, o)).astype(np.float32)
            avail = (rng.random((N, n, A)) < 0.5).astype(np.int32)
            avail[..., 0] = 1
            reset = np.zeros(N, bool)
            eps = np.full(N, 0.3)
            act = lambda: m.act(obs, avail, reset, eps)
            for _ in range(a.warmup):
                act()
            act_ms = timed(act, a.rounds)
            io = m._act_io
            dev = lambda: m.act_device(io["obs"][:N], io["avail"][:N], io["reset"][:N], io["epsilon"][:N])
            for _ in range(a.warmup):
                dev()
            dev_ms = timed(dev, a.rounds)
            x = rng.normal(size=(N, 1, 1, n, o + A + n)).astype(np.float32)

            def host():
                for e in range(N):
                    q = m.infer_actions(x[e])
                    sel.select_action(q, avail[e:e + 1], 100)
            host()
            host_ms = timed(host, a.host_rounds)
            rows.append(dict(N=N, act_ms=round(act_ms, 4), act_device_ms=round(dev_ms, 4), host_ms=round(host_ms, 4),
                             speedup=round(host_ms / act_ms, 2)))
        res[name] = dict(n_agents=n, n_actions=A, obs=o, rows=rows)
        del m
    gpu, power = card()
    res.update(gpu=gpu, power_limit=power, rnn_hidden_dim=64)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
