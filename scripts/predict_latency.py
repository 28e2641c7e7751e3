#!/usr/bin/env python
"""Host-side latency of one learner-side batched inference call (PPO, batch E): where the microseconds between
"frames in pageable host memory" and "actions back in numpy" go.  Usage: python scripts/predict_latency.py [E] [calls]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
import xingtian_b200 as xb
from xingtian_b200.capi import check
from xingtian_b200.engine import _ptr, stream_ptr

E = int(sys.argv[1]) if len(sys.argv) > 1 else 32
calls = int(sys.argv[2]) if len(sys.argv) > 2 else 300
info = {"actor": {"model_name": "PpoCnn", "state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8",
                  "model_config": {"BATCH_SIZE": 320, "LR": 0.00025, "NUM_SGD_ITER": 4, "hidden_sizes": [256],
                                   "VF_SHARE_LAYERS": True, "activation": "relu", "action_type": "Categorical"}}}
alg = xb.alg_builder("PPO", info, {"instance_num": E, "agent_num": 1})
m = alg.actor
lib = m.net.lib
rng = np.random.default_rng(0)
frames = [rng.integers(0, 256, (E, 84, 84, 4), dtype=np.uint8) for _ in range(8)]


def bench(fn, n=calls):
    for i in range(20):
        fn(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e6


rows = []
rows.append(("model.predict(state) [python + native]", bench(lambda i: m.predict(frames[i & 7]))))
m.keep_predict_obs(E, 128)
rows.append(("  .. with the device observation ring", bench(lambda i: m.predict(frames[i & 7]))))
m._obs_ring = None
io = m._predict_io(E)
off = m._offset_dev
args = lambda st: (m.net.handle, st.ctypes.data, st.nbytes, io["obs_ptr"], E, m.pi_t, m.v_t, m.ls_t, C.c_uint64(1), _ptr(off),
                   io["out_dev_ptr"], io["pin_out_ptr"], None, 1, stream_ptr())
rows.append(("xtb_ppo_predict_host alone (ctypes)", bench(lambda i: check(lib.xtb_ppo_predict_host(*args(frames[i & 7]))))))
rows.append(("staged H2D of the frames + stream sync", bench(lambda i: (
    check(lib.xtb_copy_h2d_staged(io["obs_ptr"], frames[i & 7].ctypes.data, frames[i & 7].nbytes, stream_ptr())),
    check(lib.xtb_stream_sync(stream_ptr()))))))
pin = torch.from_numpy(frames[0]).pin_memory()
rows.append(("cudaMemcpyAsync from pinned + sync (floor)", bench(lambda i: (io["obs"].copy_(pin, non_blocking=True), torch.cuda.current_stream().synchronize()))))
out_a = torch.empty(E, dtype=torch.int32, device="cuda"); out_l = torch.empty(E, device="cuda"); out_v = torch.empty(E, device="cuda")
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
graph = lambda: m.rollout_infer_device(io["obs"], None, E, 1, out_a, out_l, out_v)
for _ in range(5):
    graph()
torch.cuda.synchronize(); ev[0].record()
for _ in range(calls):
    graph()
ev[1].record(); torch.cuda.synchronize()
rows.append(("device time of the inference graph (events)", ev[0].elapsed_time(ev[1]) / calls * 1e3))
rows.append(("graph launch + sync, obs resident", bench(lambda i: (graph(), torch.cuda.current_stream().synchronize()))))
for name, us in rows:
    print("%-48s %8.1f us" % (name, us))
print("E=%d, %d bytes/call, stage threads=%s" % (E, frames[0].nbytes, os.environ.get("XTB_STAGE_THREADS", "4")))
