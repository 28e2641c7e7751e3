"""Time the graph-replayed PPO train call and the T-step rollout inference for each hidden activation, alternated in one
process: relu and tanh (the activations the engine had) against sigmoid, softsign, softplus, leaky_relu, elu, selu,
swish and gelu.  softsign, swish and gelu keep their pre-activation for the backward (include/xtb200.h), so they also
show what writing and reading it costs.

Shapes (fused heads, the default):
  c2:       PpoCnn 84x84x4 uint8 -> A = 4, [256], shared tower; E = 32 x T = 128, BATCH_SIZE 320, 4 epochs (Categorical)
  pendulum: PpoMlp [3] -> A = 1, [64, 64], separate towers; E = 10 x T = 200, BATCH_SIZE 200, 8 epochs (DiagGaussian)
Per variant and round: warm-up replays, then CUDA events around `--replays` replays of the train call and of one
rollout inference; the rounds alternate the variants.  Launches per call come from xtb_launch_count around one eager
call.  Prints the card name and power limit and one JSON line per (shape, activation) with per-round times in us.

usage: python scripts/activation_step.py [--replays 20] [--rounds 3] [--shapes c2 pendulum] [--acts relu swish ...]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from ppo_gauss_step import card, fill_rollout, make_model, train_call  # noqa: E402

ACTS = ["relu", "tanh", "sigmoid", "softsign", "softplus", "leaky_relu", "elu", "selu", "swish", "gelu"]
SHAPES = {
    "c2": dict(model="PpoCnn", state_dim=[84, 84, 4], A=4, dtype="uint8", E=32, T=128, batch=320, epochs=4,
               action_type="Categorical", cfg={"hidden_sizes": [256], "VF_SHARE_LAYERS": True}),
    "pendulum": dict(model="PpoMlp", state_dim=[3], A=1, dtype="float32", E=10, T=200, batch=200, epochs=8,
                     action_type="DiagGaussian", cfg={"hidden_sizes": [64, 64], "VF_SHARE_LAYERS": False}),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=list(SHAPES), choices=list(SHAPES))
    ap.add_argument("--acts", nargs="+", default=ACTS, choices=ACTS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("activation_step.py needs a CUDA device")
    import xingtian_b200  # noqa: F401
    from xingtian_b200 import capi
    lib = capi.lib()
    print("card: %s" % card())
    for name in args.shapes:
        base = SHAPES[name]
        E, T = base["E"], base["T"]
        variants = {}
        for act in args.acts:
            sh = dict(base, cfg=dict(base["cfg"], activation=act))
            m = make_model(sh, base["action_type"])
            N = fill_rollout(m, sh, np.random.default_rng(0))
            obs = m.rollout.obs[:N]
            step_idx = (torch.arange(E, dtype=torch.int32, device="cuda")[None, :] * T +
                        torch.arange(T, dtype=torch.int32, device="cuda")[:, None]).contiguous()
            a = torch.empty((T, E, sh["A"]) if m.gaussian else (T, E), dtype=torch.float32 if m.gaussian else torch.int32, device="cuda")
            lp, val = torch.empty(T, E, device="cuda"), torch.empty(T, E, device="cuda")
            infer = lambda m=m, obs=obs, si=step_idx, a=a, lp=lp, v=val: m.rollout_infer_device(obs, si, E, T, a, lp, v)  # noqa: E731
            variants[act] = (m, N, infer)
        launches = {}
        for act, (m, N, infer) in variants.items():
            m.use_graph = False
            got = []
            for fn in (lambda: train_call(m, N), infer):
                torch.cuda.synchronize()
                before = lib.xtb_launch_count()
                fn()
                torch.cuda.synchronize()
                got.append(int(lib.xtb_launch_count() - before))
            launches[act] = got
            m.use_graph = True
        times = {v: ([], []) for v in variants}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for act, (m, N, infer) in variants.items():
                for k, fn in enumerate((lambda: train_call(m, N), infer)):
                    for _ in range(3):
                        fn()
                    e0.record()
                    for _ in range(args.replays):
                        fn()
                    e1.record()
                    e1.synchronize()
                    times[act][k].append(e0.elapsed_time(e1) * 1e3 / args.replays)
        for act, (m, N, _) in variants.items():
            print(json.dumps({"shape": name, "act": act, "A": base["A"], "N": N, "batch": base["batch"], "epochs": base["epochs"],
                              "train_us": [round(t, 1) for t in times[act][0]], "train_launches": launches[act][0],
                              "rollout_T": T, "rollout_us": [round(t, 1) for t in times[act][1]],
                              "rollout_launches": launches[act][1], "replays": args.replays}), flush=True)
        del variants
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
