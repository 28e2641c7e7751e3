"""Time the graph-replayed DQN learner step (xtb_dqn_train) at C4 shapes for three variants, alternated in one process:
plain DqnCnn, dueling DqnCnn with the fused dueling TD step, and dueling DqnCnn layer by layer (xtb_set_fuse_heads(0)).

DqnCnn on 84x84x4 uint8 frames, B = 512 rows drawn from a 4096-transition device replay ring, A in {4, 6, 9} (A = 9 is
beyond the fused kernel's limits, so both dueling variants run layer by layer there).  Per variant and round: warm-up
replays, then CUDA events around `--replays` (default 200) graph replays; the rounds alternate the variants.  Launches
per step come from xtb_launch_count around one eager (non-graph) call.  Prints the card name and power limit and one
JSON line per (A, variant) with the per-round step times in microseconds.

usage: python scripts/dueling_step.py [--replays 200] [--rounds 3] [--actions 4 6 9]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--actions", type=int, nargs="+", default=[4, 6, 9])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dueling_step.py needs a CUDA device")
    from xingtian_b200 import capi
    from xingtian_b200.model.dqn import DqnCnn
    lib = capi.lib()
    print("card: %s" % card())
    B, ring = 512, 4096
    rng = np.random.default_rng(0)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    obs = dev(rng.integers(0, 256, (ring, 84, 84, 4), dtype=np.uint8))
    nxt = dev(rng.integers(0, 256, (ring, 84, 84, 4), dtype=np.uint8))
    rew = dev(np.sign(rng.standard_normal(ring)).astype(np.float32))
    done = dev((rng.random(ring) < 0.05).astype(np.uint8))
    idx = dev(rng.permutation(ring)[:B].astype(np.int32))
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    for A in args.actions:
        act = dev(rng.integers(0, A, ring).astype(np.int32))
        variants = {}
        for name, dueling, fuse in (("plain", False, 1), ("dueling_fused", True, 1), ("dueling_layers", True, 0)):
            mk = lambda graph: DqnCnn({"state_dim": [84, 84, 4], "action_dim": A,   # noqa: E731
                                       "model_config": {"dueling": dueling, "init_seed": 0, "use_cuda_graph": graph}})
            online, target = mk(True), mk(True)
            variants[name] = (online, target, fuse)
        step = lambda online, target: online.train_td_device(target, obs, act, rew, nxt, done, B, 0.99, loss, idx=idx)  # noqa: E731
        launches = {}
        for name, (online, target, fuse) in variants.items():
            lib.xtb_set_fuse_heads(fuse)
            online.use_graph = False
            torch.cuda.synchronize()
            before = lib.xtb_launch_count()
            step(online, target)
            torch.cuda.synchronize()
            launches[name] = int(lib.xtb_launch_count() - before)
            online.use_graph = True
            for _ in range(20):
                step(online, target)
        times = {n: [] for n in variants}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for name, (online, target, fuse) in variants.items():
                lib.xtb_set_fuse_heads(fuse)
                for _ in range(10):
                    step(online, target)
                e0.record()
                for _ in range(args.replays):
                    step(online, target)
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) * 1e3 / args.replays)
        lib.xtb_set_fuse_heads(1)
        for name in variants:
            print(json.dumps({"A": A, "variant": name, "B": B, "step_us": [round(t, 1) for t in times[name]],
                              "launches_per_step": launches[name], "replays": args.replays}))


if __name__ == "__main__":
    main()
