"""Time the graph-replayed IMPALA.train call (xtb_impala_keras_train: forward of every state, V-trace, one Keras fit
epoch per BATCH_SIZE slice) at two shapes, on the tensor-core and the fp32 kernel paths (xtb_set_tc_mode), alternated in
one process:

  cartpole: ImpalaMlp [4] -> 2, 2 trajectories x 200 steps, BATCH_SIZE 800 (examples/cartpole_impala.yaml);
  atari:    ImpalaCnn 84x84x4 uint8, 4 trajectories x 128 steps, BATCH_SIZE 512, A in {4, 18}.

Per variant and round: warm-up replays, then CUDA events around `--replays` (default 50) graph replays on the same
stored trajectories.  Launches per call come from xtb_launch_count around one eager call.  Prints the card name and
power limit and one JSON line per (shape, variant) with the per-round call times in microseconds.

usage: python scripts/impala_keras_step.py [--replays 50] [--rounds 3]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.dueling_step import card  # noqa: E402


def build(model_name, state_dim, A, L, batch, n_traj):
    import xingtian_b200 as xb
    info = {"actor": {"model_name": model_name, "state_dim": state_dim, "action_dim": A, "model_config": {"init_seed": 0}}}
    alg = xb.alg_builder("IMPALA", info, {"instance_num": 1, "agent_num": 1, "BATCH_SIZE": batch, "episode_len": L})
    rng = np.random.default_rng(0)
    for _ in range(n_traj):
        shape = (L + 1,) + tuple(state_dim)
        s = rng.integers(0, 256, shape, dtype=np.uint8) if len(state_dim) == 3 else rng.standard_normal(shape).astype(np.float32)
        alg.prepare_data(dict(cur_state=s, real_action=np.eye(A)[rng.integers(0, A, L)], action=np.full((L, A), 1.0 / A),
                              reward=rng.choice([-1.0, 0.0, 1.0], size=L).tolist(), done=(rng.random(L) < 0.01).tolist()))
    np.random.seed(0)
    alg.train()   # stages the shuffle order, sizes the net, captures the graph

    def step(graph=True):
        from xingtian_b200.algorithm import impala as mod
        from xingtian_b200.capi import ImpalaTraj, check
        from xingtian_b200.engine import _ptr, stream_ptr
        m, st, net = alg.actor, alg._store, alg.actor.net
        tr = ImpalaTraj(_ptr(st["obs"]), _ptr(st["behav"]), _ptr(st["amat"]), _ptr(st["reward"]), _ptr(st["done"]))
        check(net.lib.xtb_impala_keras_train(net.handle, m.opt.handle, tr, n_traj, L, batch, 128, _ptr(st["order"]),
                                             _ptr(st["obs_idx"]), float(mod.GAMMA), float(m.ent_coef), net.tid[m.logit_name],
                                             net.tid[m.value_name], _ptr(st["pg_adv"]), _ptr(st["tv"]), _ptr(st["loss"]),
                                             1 if graph else 0, stream_ptr()))
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("impala_keras_step.py needs a CUDA device")
    from xingtian_b200 import capi
    lib = capi.lib()
    print("card: %s" % card())
    shapes = [("cartpole", "ImpalaMlp", [4], 2, 200, 800, 2), ("atari_A4", "ImpalaCnn", [84, 84, 4], 4, 128, 512, 4),
              ("atari_A18", "ImpalaCnn", [84, 84, 4], 18, 128, 512, 4)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, model, sd, A, L, batch, n_traj in shapes:
        step = build(model, sd, A, L, batch, n_traj)
        variants = {"tensor_cores": 1, "fp32": 0}
        launches = {}
        for v, tc in variants.items():
            lib.xtb_set_tc_mode(tc)
            torch.cuda.synchronize()
            before = lib.xtb_launch_count()
            step(graph=False)
            torch.cuda.synchronize()
            launches[v] = int(lib.xtb_launch_count() - before)
            for _ in range(5):
                step()
        times = {v: [] for v in variants}
        for _ in range(args.rounds):
            for v, tc in variants.items():
                lib.xtb_set_tc_mode(tc)
                for _ in range(3):
                    step()
                e0.record()
                for _ in range(args.replays):
                    step()
                e1.record()
                e1.synchronize()
                times[v].append(e0.elapsed_time(e1) * 1e3 / args.replays)
        lib.xtb_set_tc_mode(1)
        for v in variants:
            print(json.dumps({"shape": name, "model": model, "A": A, "trajectories": n_traj, "episode_len": L, "BATCH_SIZE": batch,
                              "variant": v, "call_us": [round(t, 1) for t in times[v]], "launches_per_call": launches[v],
                              "replays": args.replays}), flush=True)


if __name__ == "__main__":
    main()
