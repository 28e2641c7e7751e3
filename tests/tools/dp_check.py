#!/usr/bin/env python
"""Data-parallel equivalence on real GPUs (run under torchrun, 2+ ranks):
every rank trains on its own env shard with gradients all-reduced over NCCL; rank 0 also trains a single-GPU
replica on the concatenated rollout with the interleaved minibatch order.  Loss traces and final weights must agree.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/tools/dp_check.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np, torch, torch.distributed as dist

rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
import xingtian_b200 as xb
from xingtian_b200 import engine
from oracle import xt_oracle as orc

E, T, BL, EPOCHS = 4, 16, 16, 2           # per rank: 64 samples, local minibatch 16
N = E * T


def make_alg(batch):
    info = {"actor": {"model_name": "PpoCnn", "state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8",
                      "device": "cuda:%d" % local,
                      "model_config": {"BATCH_SIZE": batch, "ENTROPY_LOSS": 0.003, "LOSS_CLIPPING": 0.1, "LR": 0.00025, "NUM_SGD_ITER": EPOCHS,
                                       "hidden_sizes": [256], "action_type": "Categorical", "init_seed": 11}}}
    return xb.alg_builder("PPO", info, {"instance_num": E, "agent_num": 1})


def fill(alg, shards):
    for r in shards:
        ro = orc.synth_ppo_rollout(100 + r, E, T)
        for e in range(E):
            sl = slice(e * T, (e + 1) * T)
            adv, ov, tv = orc.gae(ro["value"][e], ro["reward"][sl], ro["done"][sl])
            alg.prepare_data(dict(cur_state=ro["obs"][sl], action=ro["action"][sl], logp=ro["logp"][sl], adv=adv, old_value=ov, target_value=tv))


perms = [np.stack([np.random.default_rng(1000 * r + e).permutation(N) for e in range(EPOCHS)]).astype(np.int32) for r in range(world)]
# ---- data-parallel run
dp_first = None
alg = make_alg(BL)
dp = engine.GradComm()
fill(alg, [rank])
loss_dp = alg.actor.train_device(N, perm=perms[rank])
trace_dp = torch.tensor(alg.actor.last_losses, device="cuda")
dist.all_reduce(trace_dp)                      # per-rank losses are partial sums of the global mean
w_dp = np.concatenate([v.ravel() for v in alg.get_weights().values()])
print('rank %d: dp run done' % rank, flush=True)
dp.detach()
# weights identical on every rank
wt = torch.from_numpy(w_dp).cuda(); w0 = wt.clone(); dist.broadcast(w0, 0)
assert torch.equal(wt, w0), "replicas diverged"
if rank == 0:
    ref = make_alg(BL * world)
    fill(ref, list(range(world)))
    steps = N // BL
    perm = np.concatenate([np.concatenate([perms[r][e, s * BL:(s + 1) * BL] + r * N for r in range(world)]) for e in range(EPOCHS) for s in range(steps)]).astype(np.int32)
    ref.actor.train_device(N * world, perm=perm.reshape(EPOCHS, -1))
    w_ref = np.concatenate([v.ravel() for v in ref.get_weights().values()])
    w_init = np.concatenate([v.ravel() for v in make_alg(BL).get_weights().values()])
    tr = trace_dp.cpu().numpy(); tr_ref = ref.actor.last_losses
    err_t = np.max(np.abs(tr - tr_ref)) / np.max(np.abs(tr_ref))
    err_w = np.linalg.norm((w_dp - w_init) - (w_ref - w_init)) / np.linalg.norm(w_ref - w_init)
    print("DP check world=%d: loss-trace rel err %.2e, weight-update l2 rel err %.2e" % (world, err_t, err_w))
    ok = err_t < 5e-3 and err_w < 5e-2
    print("DP_CHECK_OK" if ok else "DP_CHECK_FAILED", flush=True)
    sys.stdout.flush()
    os._exit(0 if ok else 1)
sys.stdout.flush()
os._exit(0)
