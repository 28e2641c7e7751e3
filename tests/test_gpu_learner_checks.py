"""Argument checks the learner entry points share: xtb_impala_train and xtb_dqn_train, like xtb_ppo_train, refuse an
optimiser sized for another parameter count before they launch anything, eagerly or graphed."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_plugins import alg_cfg

pytestmark = pytest.mark.gpu

XTB_ERR_ARG = -1


def _optimiser_of_size(lib, capi, n):
    from xingtian_b200.engine import _ptr
    mom, var = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    seg = (C.c_longlong * 2)(0, n)
    opt = C.c_void_p()
    capi.check(lib.xtb_adam_create(n, 2.5e-4, 0.9, 0.999, 1e-8, capi.CLIP_GLOBAL_NORM, 5.0, seg, 1, _ptr(mom), _ptr(var),
                                   C.byref(opt)))
    return opt, (mom, var)


def _assert_refused(lib, call):
    for use_graph in (0, 1):
        torch.cuda.synchronize()
        n0 = lib.xtb_launch_count()
        assert call(use_graph) == XTB_ERR_ARG
        assert b"size mismatch" in lib.xtb_last_error()
        assert lib.xtb_launch_count() == n0


def test_impala_train_rejects_optimiser_of_another_size():
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = capi.lib()
    S, n = 16, 32
    info = {"actor": {"model_name": "ImpalaCnnOpt", "state_dim": [84, 84, 4], "input_dtype": "uint8", "state_mean": 0.0,
                      "state_std": 255.0, "action_dim": 4,
                      "model_config": {"LR": 0.0005, "sample_batch_step": S, "grad_norm_clip": 40.0, "init_seed": 3}}}
    m = xb.alg_builder("IMPALAOpt", info, alg_cfg(instance_num=2, prepare_times_per_train=1, BATCH_SIZE=n)).actor
    net = m.net
    net.ensure_batch(n)
    obs = torch.zeros(n, 84, 84, 4, dtype=torch.uint8, device="cuda")
    bp_logits = torch.zeros(n, 4, device="cuda")
    action = torch.zeros(n, dtype=torch.int32, device="cuda")
    done = torch.zeros(n, dtype=torch.uint8, device="cuda")
    reward = torch.zeros(n, device="cuda")
    loss = torch.zeros(1, device="cuda")
    opt, _keep = _optimiser_of_size(lib, capi, net.n_params - 1)
    try:
        _assert_refused(lib, lambda use_graph: lib.xtb_impala_train(
            net.handle, opt, _ptr(obs), None, _ptr(bp_logits), _ptr(action), _ptr(done), _ptr(reward), n, S, 0.99,
            net.tid[m.logit_name], net.tid[m.base_name], _ptr(loss), use_graph, stream_ptr()))
    finally:
        lib.xtb_adam_destroy(opt)


def test_dqn_train_rejects_optimiser_of_another_size():
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = capi.lib()
    info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": 4, "model_config": {"LR": 0.00015, "init_seed": 5}}}
    alg = xb.alg_builder("DQN", info, alg_cfg(instance_num=1, learning_starts=8, BUFFER_SIZE=64, BATCH_SIZE=32))
    m, tgt = alg.actor, alg.target_actor
    n, A = 32, 4
    rng = np.random.default_rng(2)
    obs = torch.from_numpy(rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)).cuda()
    next_obs = torch.from_numpy(rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)).cuda()
    action = torch.zeros(n, dtype=torch.int32, device="cuda")
    reward = torch.zeros(n, device="cuda")
    done = torch.zeros(n, dtype=torch.uint8, device="cuda")
    qn_t = torch.empty(n, A, device="cuda")
    loss = torch.zeros(1, device="cuda")
    opt, _keep = _optimiser_of_size(lib, capi, m.net.n_params - 1)
    try:
        _assert_refused(lib, lambda use_graph: lib.xtb_dqn_train(
            m.net.handle, tgt.net.handle, opt, _ptr(obs), _ptr(next_obs), None, _ptr(action), _ptr(reward), _ptr(done), None, n,
            0.99, 0.0, m.net.tid[m.q_name], _ptr(qn_t), None, _ptr(loss), use_graph, stream_ptr()))
    finally:
        lib.xtb_adam_destroy(opt)
