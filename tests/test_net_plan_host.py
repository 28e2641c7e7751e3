"""CPU tier: xtb_net_create plans a network on the host and makes no CUDA call, so every shipped architecture can be
planned without a GPU.  Each plan (every xtb_layer_plan field, xtb_net_layer_params and the parameter count) is pinned
to the table below; a descriptor rejected after an accepted conv layer reports its error."""
import ctypes as C

import pytest

from xingtian_b200.engine import net_desc
from xingtian_b200.model import archs


@pytest.fixture(scope="module")
def lib():
    from xingtian_b200 import build, capi
    build.build()
    return capi.lib()


def _conv(name, src, k, s, cout, pad):
    return (name, "conv", src, dict(k=k, s=s, cout=cout, pad=pad, act="tanh"))


def _large_map(hw):
    """test_large_map_conv_falls_back's net: an s2d stem, then a 3x3 SAME 32 -> 32 conv on an hw map"""
    return dict(input_dtype="uint8", state_dim=(4 * hw, 4 * hw, 4), scale=1.0 / 255.0,
                layers=[_conv("x", "obs", 4, 4, 32, "valid"), _conv("y", "x", 3, 1, 32, "same")], outputs=["y"])


# MuzeroCnn at its default supports (value 0..60000: 305, reward -300..300: 26) and unroll 5: prediction runs 6 x 256 rows
_MZ = archs.muzero_cnn((84, 84, 4), 4, 305, 26)
ARCHS = {
    "ppo_cnn@320": (archs.ppo_cnn((84, 84, 4), 4, [256], "relu", True), 320),
    "ppo_cnn@512": (archs.ppo_cnn((84, 84, 4), 4, [256], "relu", True), 512),
    "ppo_cnn@4096": (archs.ppo_cnn((84, 84, 4), 4, [256], "relu", True), 4096),
    "impala_cnn@512": (archs.impala_cnn((84, 84, 4), 4), 512),
    "dqn_cnn@512": (archs.dqn_cnn((84, 84, 4), 4), 512),
    "dqn_cnn_dueling@512": (archs.dqn_cnn((84, 84, 4), 4, dueling=True), 512),
    "impala_keras_cnn@512": (archs.impala_keras_cnn((84, 84, 4), 4), 512),
    "muzero_rep@256": (_MZ[0], 256),
    "muzero_dyn@256": (_MZ[1], 256),
    "muzero_pred@1536": (_MZ[2], 1536),
    "ppo_mlp@512": (archs.ppo_mlp((4,), 2, [64, 64], "tanh", False), 512),
    "large_map_42@9": (_large_map(42), 9),
    "large_map_24@9": (_large_map(24), 9),
}

# parameter count, then per layer: kind, tc, s2d, w_res, n_fwd, n_dg, R, fwd_stages, dg_stages, dg_empty_units, k_slices
# (xtb_layer_plan), kernel_off, bias_off, k_rows, n_cols (xtb_net_layer_params)
_PPO_CONV = [(0, 1, 1, 1, 32, 64, 2, 4, 4, 0, 1, 0, 8192, 256, 32),
             (0, 1, 0, 1, 32, 32, 4, 4, 4, 0, 1, 8224, 24608, 512, 32),
             (0, 1, 0, 1, 64, 32, 3, 4, 4, 0, 1, 24640, 43072, 288, 64)]
_PPO_HEADS = [(1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 846208, 847232, 256, 4),
              (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 847236, 847492, 256, 1)]
_DQN_TRUNK = [(0, 1, 1, 1, 32, 64, 2, 4, 4, 0, 1, 0, 8192, 256, 32),
              (0, 1, 0, 0, 64, 32, 4, 4, 4, 0, 1, 8224, 40992, 512, 64),
              (0, 1, 0, 0, 64, 64, 6, 4, 3, 0, 1, 41056, 77920, 576, 64),
              (1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 7, 77984, 880800, 3136, 256),
              (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 881056, 882080, 256, 4)]
_STEM = (0, 1, 1, 1, 32, 64, 1, 4, 4, 0, 1, 0, 2048, 64, 32)
PLANS = {
    "ppo_cnn@320": (847493, _PPO_CONV + [(1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 10, 43136, 845952, 3136, 256)] + _PPO_HEADS),
    "ppo_cnn@512": (847493, _PPO_CONV + [(1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 7, 43136, 845952, 3136, 256)] + _PPO_HEADS),
    "ppo_cnn@4096": (847493, _PPO_CONV + [(1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 1, 43136, 845952, 3136, 256)] + _PPO_HEADS),
    "impala_cnn@512": (1005109, [(0, 1, 1, 1, 16, 64, 2, 4, 4, 0, 1, 0, 4096, 256, 16),
                                 (0, 1, 0, 1, 32, 16, 4, 4, 4, 0, 1, 4112, 12304, 256, 32),
                                 (1, 1, 0, 0, 64, 32, 0, 4, 4, 0, 8, 12336, 1003568, 3872, 256),
                                 (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1003824, 1004848, 256, 4),
                                 (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1004852, 1005108, 256, 1)]),
    "dqn_cnn@512": (882084, _DQN_TRUNK),
    "dqn_cnn_dueling@512": (882341, _DQN_TRUNK + [(1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 882084, 882340, 256, 1),
                                                  (2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 882341, 882341, 0, 0)]),
    "impala_keras_cnn@512": (882341, _DQN_TRUNK + [(1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 882084, 882340, 256, 1)]),
    "muzero_rep@256": (846208, _PPO_CONV + [(1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 13, 43136, 845952, 3136, 256)]),
    "muzero_dyn@256": (136090, [(1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 66560, 260, 256),
                                (1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 4, 66816, 99584, 256, 128),
                                (1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 1, 99712, 132480, 128, 256),
                                (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 132736, 136064, 128, 26)]),
    "muzero_pred@1536": (72757, [(1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 32768, 256, 128),
                                 (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 32896, 33408, 128, 4),
                                 (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 33412, 72452, 128, 305)]),
    "ppo_mlp@512": (9155, [(1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 256, 4, 64),
                           (1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 1, 320, 4416, 64, 64),
                           (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4480, 4736, 4, 64),
                           (1, 1, 0, 0, 64, 64, 0, 4, 3, 0, 1, 4800, 8896, 64, 64),
                           (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 8960, 9088, 64, 2),
                           (1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 9090, 9154, 64, 1)]),
    "large_map_42@9": (11328, [_STEM, (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2080, 11296, 288, 32)]),
    "large_map_24@9": (11328, [_STEM, (0, 1, 0, 1, 32, 32, 3, 4, 3, 0, 1, 2080, 11296, 288, 32)]),
}


def _create(lib, arch, max_batch):
    h = C.c_void_p()
    rc = lib.xtb_net_create(C.byref(net_desc(arch)), max_batch, C.byref(h))
    return rc, h


@pytest.mark.parametrize("case", list(ARCHS))
def test_shipped_architectures_plan_on_the_host(lib, case):
    from xingtian_b200 import capi
    arch, max_batch = ARCHS[case]
    launches = lib.xtb_launch_count()
    rc, h = _create(lib, arch, max_batch)
    assert rc == 0, lib.xtb_last_error()
    try:
        got = []
        for i in range(len(arch["layers"])):
            p = capi.LayerPlan()
            assert lib.xtb_net_layer_plan(h, i, C.byref(p)) == 0
            ko, bo, kr, nc = C.c_longlong(), C.c_longlong(), C.c_int(), C.c_int()
            assert lib.xtb_net_layer_params(h, i, C.byref(ko), C.byref(bo), C.byref(kr), C.byref(nc)) == 0
            got.append(tuple(getattr(p, f) for f, _ in capi.LayerPlan._fields_) + (ko.value, bo.value, kr.value, nc.value))
        assert (lib.xtb_net_param_count(h), got) == PLANS[case]
        assert lib.xtb_net_workspace_bytes(h) > 0
    finally:
        lib.xtb_net_destroy(h)
    assert lib.xtb_launch_count() == launches


def test_layer_rejected_after_a_conv_layer(lib):
    arch = dict(input_dtype="uint8", state_dim=(84, 84, 4), scale=1.0 / 255.0,
                layers=[_conv("a", "obs", 8, 4, 32, "valid"), _conv("b", "a", 3, 3, 32, "valid")], outputs=["b"])
    rc, h = _create(lib, arch, 32)
    assert rc == -1 and not h.value                                  # XTB_ERR_ARG
    assert b"layer 1: stride must be 1,2,4" in lib.xtb_last_error(), lib.xtb_last_error()
