"""Prioritized replay against uniform replay for the DQN step: DqnCnn at the C4 shape (B = 512, 84x84x4 uint8 frames, 4
actions) over a full ring of 2^16 and of 400 000 slots (sum-tree depth 19).

Per ring it reports
  - the time per training step as DQN.train runs it, ending in the loss read that synchronises:
      uniform:     host random.sample + index copy + the xtb_dqn_train graph
      prioritized: the xtb_dqn_per_train graph (draw + weighted step + priority update) + the status read
  - the sample and update kernels alone (xtb_per_sample with Philox, xtb_per_update), CUDA events over many launches;
and the card's name and power limit, read in the same run.  One JSON object on stdout (and in --out when given).

    python scripts/dqn_per_step.py --steps 200 --warmup 20
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power)
    except Exception as err:      # no nvidia-smi: the name from the runtime, the power limit unknown
        return dict(name=torch.cuda.get_device_name(0), power_limit="unknown (%s)" % err)


def events_ms(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def run_ring(ring, B, steps, warmup, launches):
    import ctypes as C
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    from xingtian_b200.model.dqn import DqnCnn
    lib = capi.lib()
    A = 4
    mk = lambda: DqnCnn({"state_dim": [84, 84, 4], "action_dim": A, "max_batch": B,   # noqa: E731
                         "model_config": {"init_seed": 1, "LR": 0.00015}})
    uni, per_model, tgt = mk(), mk(), mk()
    g = torch.Generator(device="cuda").manual_seed(ring)
    obs = torch.randint(0, 256, (ring, 84, 84, 4), dtype=torch.uint8, device="cuda", generator=g)
    nxt = torch.randint(0, 256, (ring, 84, 84, 4), dtype=torch.uint8, device="cuda", generator=g)
    act = torch.randint(0, A, (ring,), dtype=torch.int32, device="cuda", generator=g)
    rew = torch.randn(ring, device="cuda", generator=g)
    done = (torch.rand(ring, device="cuda", generator=g) < 0.01).to(torch.uint8)
    h = C.c_void_p()
    capi.check(lib.xtb_per_create(ring, 0.6, 1e-6, 12345, C.byref(h)))
    capi.check(lib.xtb_per_add(h, 0, ring, stream_ptr()))
    loss = torch.zeros(1, device="cuda")
    idx_dev = torch.zeros(B, dtype=torch.int32, device="cuda")
    p_idx, p_w, p_td = (torch.zeros(B, dtype=dt, device="cuda") for dt in (torch.int32, torch.float32, torch.float32))
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    random.seed(0)

    def uniform_step():
        picks = np.asarray(random.sample(range(ring), B), np.int32)
        idx_dev.copy_(torch.from_numpy(picks))
        uni.train_td_device(tgt, obs, act, rew, nxt, done, B, 0.99, loss, idx=idx_dev)
        return float(loss.cpu()[0])

    def per_step():
        per_model.train_per_device(tgt, h, 0.4, obs, act, rew, nxt, done, B, 0.99, loss, p_idx, p_w, p_td, status)
        out = float(loss.cpu()[0])
        assert int(status.cpu()[0]) == 0
        return out

    res = {}
    for name, fn in (("uniform", uniform_step), ("prioritized", per_step), ("uniform_again", uniform_step),
                     ("prioritized_again", per_step)):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        res[name + "_step_ms"] = (time.perf_counter() - t0) * 1e3 / steps
    sidx, sw = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, device="cuda")
    td = torch.rand(B, device="cuda", generator=g)
    uidx = torch.randint(0, ring, (B,), dtype=torch.int32, device="cuda", generator=g)
    st = stream_ptr()
    sample = lambda: lib.xtb_per_sample(h, B, 0.4, None, _ptr(sidx), _ptr(sw), st)   # noqa: E731
    update = lambda: lib.xtb_per_update(h, _ptr(uidx), _ptr(td), B, st)              # noqa: E731
    for fn in (sample, update):
        for _ in range(20):
            capi.check(fn())
    res["sample_kernel_us"] = events_ms(sample, launches) * 1e3
    res["update_kernel_us"] = events_ms(update, launches) * 1e3
    lib.xtb_per_destroy(h)
    del obs, nxt
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--rings", default="65536,400000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dqn_per_step: needs a CUDA device")
    from xingtian_b200 import build
    build.build()
    out = dict(card=card(), batch=args.batch, steps=args.steps, warmup=args.warmup, launches=args.launches, rings={})
    for ring in [int(x) for x in args.rings.split(",")]:
        out["rings"][str(ring)] = run_ring(ring, args.batch, args.steps, args.warmup, args.launches)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
