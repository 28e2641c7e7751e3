"""Time the graph-replayed PPO train call (xtb_ppo_train) and rollout inference (xtb_ppo_rollout_infer) of a
DiagGaussian actor against a Categorical one with the same network, alternated in one process.

Shapes:
  pendulum: PpoMlp [3] -> A = 1, tanh [64, 64], separate towers; E = 10 envs x T = 200 steps, BATCH_SIZE 200, 8 epochs
  pixel:    PpoCnn 84x84x4 uint8 -> A = 3, relu [256], shared tower; E = 32 x T = 128, BATCH_SIZE 320, 4 epochs
Variants: gauss_fused (the fused Gaussian heads: heads_kernel<PpoGaussLoss> in training, infer_heads_kernel<DiagGaussian> in
inference; the default), gauss_layers (xtb_set_fuse_heads(0)), and the same two for Categorical at the same A.  Per variant and round: warm-up
replays, then CUDA events around `--replays` graph replays of the train call and of one T-step rollout inference; the
rounds alternate the variants.  Launches per call come from xtb_launch_count around one eager (non-graph) call.  Prints
the card name and power limit and one JSON line per (shape, variant) with per-round times in microseconds.

usage: python scripts/ppo_gauss_step.py [--replays 30] [--rounds 3] [--shapes pendulum pixel]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {
    "pendulum": dict(model="PpoMlp", state_dim=[3], A=1, dtype="float32", E=10, T=200, batch=200, epochs=8,
                     cfg={"hidden_sizes": [64, 64], "activation": "tanh", "VF_SHARE_LAYERS": False}),
    "pixel": dict(model="PpoCnn", state_dim=[84, 84, 4], A=3, dtype="uint8", E=32, T=128, batch=320, epochs=4,
                  cfg={"hidden_sizes": [256], "activation": "relu", "VF_SHARE_LAYERS": True}),
}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def make_model(sh, action_type):
    from xingtian_b200.registry import Registers
    cfg = dict(sh["cfg"], BATCH_SIZE=sh["batch"], NUM_SGD_ITER=sh["epochs"], action_type=action_type, init_seed=0,
               ENTROPY_LOSS=0.01, max_predict_batch=sh["E"])
    return Registers.model[sh["model"]]({"state_dim": sh["state_dim"], "action_dim": sh["A"], "input_dtype": sh["dtype"],
                                         "model_config": cfg})


def fill_rollout(m, sh, rng):
    N = sh["E"] * sh["T"]
    sd = tuple(sh["state_dim"])
    obs = rng.integers(0, 256, (N,) + sd, dtype=np.uint8) if sh["dtype"] == "uint8" else rng.standard_normal((N,) + sd).astype(np.float32)
    act = rng.standard_normal((N, sh["A"])).astype(np.float32) if m.gaussian else rng.integers(0, sh["A"], N).astype(np.int32)
    lab = [act] + [rng.standard_normal(N).astype(np.float32) * s for s in (0.3, 1.0, 1.0, 1.0)]
    lab[1] = lab[1] - 1.5
    m.train([obs], lab)          # uploads the rollout, sets up the order / loss buffers, captures the graph
    return N


def train_call(m, N):
    """the native train call train_device makes, without its loss read-back"""
    lib, ro = m.net.lib, m.rollout.as_struct()
    rc = lib.xtb_ppo_train(m.net.handle, m.opt.handle, C.byref(ro), N, int(m._batch_size), int(m.num_sgd_iter),
                           C.c_void_p(m._perm_dev.data_ptr()), C.byref(m.hyper), m.pi_t, m.v_t, m.ls_t,
                           C.c_void_p(m._loss_dev.data_ptr()), 1 if m.use_graph else 0,
                           C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, lib.xtb_last_error()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=list(SHAPES), choices=list(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ppo_gauss_step.py needs a CUDA device")
    import xingtian_b200  # noqa: F401
    from xingtian_b200 import capi
    lib = capi.lib()
    print("card: %s" % card())
    for name in args.shapes:
        sh = SHAPES[name]
        rng = np.random.default_rng(0)
        E, T = sh["E"], sh["T"]
        variants = {}
        for vname, atype, fuse in (("gauss_fused", "DiagGaussian", 1), ("gauss_layers", "DiagGaussian", 0),
                                   ("cat_fused", "Categorical", 1), ("cat_layers", "Categorical", 0)):
            lib.xtb_set_fuse_heads(fuse)
            m = make_model(sh, atype)
            N = fill_rollout(m, sh, rng)
            obs = m.rollout.obs[:N]
            step_idx = (torch.arange(E, dtype=torch.int32, device="cuda")[None, :] * T +
                        torch.arange(T, dtype=torch.int32, device="cuda")[:, None]).contiguous()
            act = torch.empty((T, E, sh["A"]) if m.gaussian else (T, E), dtype=torch.float32 if m.gaussian else torch.int32, device="cuda")
            lp, val = torch.empty(T, E, device="cuda"), torch.empty(T, E, device="cuda")
            infer = lambda m=m, obs=obs, si=step_idx, a=act, lp=lp, v=val: m.rollout_infer_device(obs, si, E, T, a, lp, v)  # noqa: E731
            variants[vname] = (m, N, fuse, infer)
        launches = {}
        for vname, (m, N, fuse, infer) in variants.items():
            lib.xtb_set_fuse_heads(fuse)
            m.use_graph = False
            got = []
            for fn in (lambda: train_call(m, N), infer):
                torch.cuda.synchronize()
                before = lib.xtb_launch_count()
                fn()
                torch.cuda.synchronize()
                got.append(int(lib.xtb_launch_count() - before))
            launches[vname] = got
            m.use_graph = True
        times = {v: ([], []) for v in variants}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for vname, (m, N, fuse, infer) in variants.items():
                lib.xtb_set_fuse_heads(fuse)
                for k, fn in enumerate((lambda: train_call(m, N), infer)):
                    for _ in range(5):
                        fn()
                    e0.record()
                    for _ in range(args.replays):
                        fn()
                    e1.record()
                    e1.synchronize()
                    times[vname][k].append(e0.elapsed_time(e1) * 1e3 / args.replays)
        lib.xtb_set_fuse_heads(1)
        for vname, (m, N, _, _) in variants.items():
            print(json.dumps({"shape": name, "variant": vname, "A": sh["A"], "N": N, "batch": sh["batch"], "epochs": sh["epochs"],
                              "train_us": [round(t, 1) for t in times[vname][0]], "train_launches": launches[vname][0],
                              "rollout_T": T, "rollout_us": [round(t, 1) for t in times[vname][1]],
                              "rollout_launches": launches[vname][1], "replays": args.replays}))


if __name__ == "__main__":
    main()
