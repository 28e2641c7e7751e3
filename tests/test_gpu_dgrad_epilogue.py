"""The data-gradient epilogue reads act' and, when it accumulates, the output planes from shared memory: the producer
warp of bp_rows_kernel<2> prefetches them per tile into one of two banks guarded by full / empty mbarriers.  These cases
cover what that adds to the layer sweep: gradient rows in [B, round16(B)) that must stay zero, launches whose CTAs run
many tiles (both banks wrap their barrier phases many times, relu / tanh, with and without `accumulate`, against the
fp32 CUDA-core path), and bitwise reproducibility of a PPO train call."""
import numpy as np
import pytest

from oracle import xt_oracle as orc
from test_gpu_kernels import RELU_FLIP_TC, TC_GRAD_BOUND, l2_rel, xb  # noqa: F401
from test_gpu_layer_sweep import _check_parity, _conv, _gpu_run, _inputs, _plan, _weights

pytestmark = pytest.mark.gpu


def _ppo_trunk(act, accumulate):
    """PpoCnn's first two convs: uint8 84 x 84 x 4 -> x (k8 s4, 20 x 20 x 32, s2d) -> y (k4 s2, 9 x 9 x 64).  y's data
    gradient into x is 400 units x ceil(B / 128) tiles.  accumulate: a second tensor-core conv z (1 x 1, 16) reads x;
    the backward pass runs z first, so y's data gradient adds to what z wrote."""
    layers = [_conv("x", "obs", 8, 4, 32, "valid", act), _conv("y", "x", 4, 2, 64, "valid", act)]
    outputs = ["y"]
    if accumulate:
        layers.append(_conv("z", "x", 1, 1, 16, "valid", act))
        outputs.append("z")
    return dict(input_dtype="uint8", state_dim=(84, 84, 4), scale=1.0 / 255.0, layers=layers, outputs=outputs)


def _run(arch, w, B, seed=3):
    from xingtian_b200.engine import Net
    net = Net(arch, max_batch=B)
    plan = _plan(net, arch)
    net.set_weights(w)
    obs, idx, gh = _inputs(arch, B, False, seed=seed)
    return plan, obs, gh, _gpu_run(net, arch, obs, idx, B, gh)


@pytest.mark.parametrize("B", [1, 17, 129, 320])
def test_pad_rows_stay_zero(xb, B):
    """Rows [B, round16(B)) of the gradient planes are read by the weight-gradient K loop.  A pass at B + 16 leaves
    non-zero gradients there; a following pass at B on the same net must give what a fresh net gives: bit for bit where
    the fresh net reproduces itself, else within the layer sweep's float64 bounds (the top layer's bias gradient is a
    column sum whose order may vary between runs)."""
    from xingtian_b200.engine import Net
    arch = _ppo_trunk("relu", False)
    w = _weights(arch)
    used = Net(arch, max_batch=B + 16)
    used.set_weights(w)
    assert all(p["tc"] for p in _plan(used, arch).values())
    obs, idx, gh = _inputs(arch, B + 16, False, seed=7)
    _gpu_run(used, arch, obs, idx, B + 16, gh)
    obs, idx, gh = _inputs(arch, B, False, seed=8)
    got = _gpu_run(used, arch, obs, idx, B, gh)
    fresh = Net(arch, max_batch=B + 16)
    fresh.set_weights(w)
    ref1 = _gpu_run(fresh, arch, obs, idx, B, gh)
    ref2 = _gpu_run(fresh, arch, obs, idx, B, gh)
    for k in got[1]:
        if np.array_equal(ref1[1][k], ref2[1][k]):
            np.testing.assert_array_equal(got[1][k], ref1[1][k], err_msg=k)
    _check_parity("dgrad_epilogue/pad_rows/B%d" % B, arch, w, obs, idx, gh, got[0], got[1], True)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("B", [320, 4096])
def test_many_tiles_per_cta_match_fp32(xb, B, act, accumulate):
    """y's data gradient at B = 320 runs ~9 tiles per CTA, at B = 4096 ~97: the epilogue banks cycle their phases many
    times.  Every parameter gradient on the tensor cores against the fp32 kernels (ReLU: plus the slack of mask flips at
    bf16x3 forward error); at B = 320 also against float64 with the layer sweep's bounds."""
    lib = xb["lib"]
    arch = _ppo_trunk(act, accumulate)
    w = _weights(arch)
    old = lib.xtb_get_tc_mode()
    try:
        lib.xtb_set_tc_mode(1)
        plan, obs, gh, (tc_t, tc_g) = _run(arch, w, B)
        assert all(p["tc"] for p in plan.values()), plan
        lib.xtb_set_tc_mode(0)
        f32_g = _run(arch, w, B)[3][1]
    finally:
        lib.xtb_set_tc_mode(old)
    bound = TC_GRAD_BOUND + (RELU_FLIP_TC if act == "relu" else 0.0)
    bad = {k: l2_rel(tc_g[k], f32_g[k]) for k in tc_g}
    bad = {k: e for k, e in bad.items() if not e < bound}
    assert not bad, bad
    if B == 320:
        _check_parity("dgrad_epilogue/%s/%s/B%d" % (act, "acc" if accumulate else "noacc", B), arch, w, obs, None, gh,
                      tc_t, tc_g, True)


def test_ppo_train_is_bitwise_reproducible(xb):
    """Two PpoCnn train calls (320-sample minibatches, two SGD epochs) from the same weights and data agree bit for bit."""
    pkg = xb["pkg"]

    def run():
        info = {"actor": {"model_name": "PpoCnn", "state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8",
                          "model_config": {"BATCH_SIZE": 320, "ENTROPY_LOSS": 0.003, "LOSS_CLIPPING": 0.1, "LR": 0.00025,
                                           "NUM_SGD_ITER": 2, "hidden_sizes": [256], "action_type": "Categorical",
                                           "init_seed": 0}}}
        alg = pkg.alg_builder("PPO", info, {"instance_num": 8, "agent_num": 1})
        ro = orc.synth_ppo_rollout(0, 8, 80)
        for e in range(8):
            sl = slice(e * 80, (e + 1) * 80)
            alg.prepare_data(dict(cur_state=ro["obs"][sl], action=ro["action"][sl], logp=ro["logp"][sl],
                                  value=ro["value"][e], reward=ro["reward"][sl], done=ro["done"][sl]))
        np.random.seed(0)
        loss = alg.train()
        return loss, alg.get_weights()
    l1, w1 = run()
    l2, w2 = run()
    assert np.float32(l1).tobytes() == np.float32(l2).tobytes(), (l1, l2)
    for k in w1:
        np.testing.assert_array_equal(w1[k], w2[k], err_msg=k)
