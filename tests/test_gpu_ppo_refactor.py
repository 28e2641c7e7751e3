"""Contract details of the Categorical PPO entry points that share the DiagGaussian code path: rollout inference
without a step index reads the observation rows of each step, and xtb_ppo_train checks the optimiser's size before it
launches anything."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_plugins import alg_cfg, ppo_cnn_info

pytestmark = pytest.mark.gpu

XTB_ERR_ARG = -1


@pytest.mark.parametrize("fuse_heads", [1, 0])
def test_rollout_infer_without_step_idx_reads_each_steps_rows(fuse_heads):
    """step_idx = NULL: step t reads observation rows t*n_env ..; the draws, log-probs and values equal those of
    step_idx[t][e] = t*n_env + e from the same Philox offset."""
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    lib = capi.lib()
    m = xb.alg_builder("PPO", ppo_cnn_info(), alg_cfg()).actor
    E, T = 8, 3
    obs = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (T * E, 84, 84, 4), dtype=np.uint8)).cuda()
    step_idx = torch.arange(T * E, dtype=torch.int32, device="cuda")
    m._offset_dev = torch.zeros(1, dtype=torch.int64, device="cuda")

    def run(idx):
        act = torch.empty(T, E, dtype=torch.int32, device="cuda")
        lp = torch.empty(T, E, device="cuda")
        val = torch.empty(T, E, device="cuda")
        m._offset_dev.fill_(11)        # every call advances the counter by n_step
        m.rollout_infer_device(obs, idx, E, T, act, lp, val)
        torch.cuda.synchronize()
        return act.cpu().numpy(), lp.cpu().numpy(), val.cpu().numpy()

    try:
        lib.xtb_set_fuse_heads(fuse_heads)
        act_i, lp_i, val_i = run(step_idx)
        act_n, lp_n, val_n = run(None)
    finally:
        lib.xtb_set_fuse_heads(1)
    assert not np.array_equal(val_i[0], val_i[1])     # the steps see different observations
    np.testing.assert_array_equal(act_n, act_i)
    np.testing.assert_array_equal(lp_n, lp_i)
    np.testing.assert_array_equal(val_n, val_i)


def test_categorical_ppo_train_rejects_optimiser_of_another_size():
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = capi.lib()
    m = xb.alg_builder("PPO", ppo_cnn_info(), alg_cfg()).actor
    N = 24
    m.net.ensure_batch(N)
    obs = torch.zeros(N, 84, 84, 4, dtype=torch.uint8, device="cuda")
    action = torch.zeros(N, dtype=torch.int32, device="cuda")
    f = [torch.zeros(N, device="cuda") for _ in range(4)]
    ro = capi.PpoRollout(_ptr(obs), _ptr(action), *[_ptr(x) for x in f])
    perm = torch.arange(N, dtype=torch.int32, device="cuda")
    loss = torch.zeros(1, device="cuda")
    n = m.net.n_params - 1
    mom, var = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    seg = (C.c_longlong * 2)(0, n)
    opt = C.c_void_p()
    capi.check(lib.xtb_adam_create(n, 2.5e-4, 0.9, 0.999, 1e-8, capi.CLIP_GLOBAL_NORM, 5.0, seg, 1, _ptr(mom), _ptr(var),
                                   C.byref(opt)))
    try:
        for use_graph in (0, 1):
            torch.cuda.synchronize()
            n0 = lib.xtb_launch_count()
            rc = lib.xtb_ppo_train(m.net.handle, opt, C.byref(ro), N, N, 1, _ptr(perm), C.byref(m.hyper), m.pi_t, m.v_t, 0,
                                   _ptr(loss), use_graph, stream_ptr())
            assert rc == XTB_ERR_ARG
            assert b"size mismatch" in lib.xtb_last_error()
            assert lib.xtb_launch_count() == n0
    finally:
        lib.xtb_adam_destroy(opt)
