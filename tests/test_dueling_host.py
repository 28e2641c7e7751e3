"""The dueling Q head of DqnCnn / DqnMlp without a GPU: layer tables, parameter names / shapes / counts, the oracle's
combine against the reference's own layer_normalize / layer_add (tests/golden/dueling.npz) and its gradient."""
import os

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from xingtian_b200.model import archs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dueling.npz")

CNN_NAMES = ["conv2d/kernel", "conv2d/bias", "conv2d_1/kernel", "conv2d_1/bias", "conv2d_2/kernel", "conv2d_2/bias",
             "dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias", "dense_2/kernel", "dense_2/bias"]


def _pshapes(arch):
    return list(orc.param_shapes(arch).items())


@pytest.mark.parametrize("A", [4, 18])
def test_dqn_cnn_dueling_parameters(A):
    arch = archs.dqn_cnn((84, 84, 4), A, dueling=True)
    shapes = _pshapes(arch)
    assert [n for n, _ in shapes] == CNN_NAMES
    assert dict(shapes)["dense_1/kernel"] == (256, A) and dict(shapes)["dense_2/kernel"] == (256, 1)
    assert dict(shapes)["dense_2/bias"] == (1,)
    assert _pshapes(orc.dqn_cnn_arch(action_dim=A, dueling=True)) == shapes
    assert arch["outputs"] == ["dueling"]
    assert arch["layers"][-1] == ("dueling", "dueling", ("dense_1", "dense_2"), {})
    assert arch["layers"][-2][2] == "dense"
    count = sum(int(np.prod(s)) for _, s in shapes)
    if A == 4:
        assert count == 882341
    assert count == sum(int(np.prod(s)) for s in orc.param_shapes(orc.dqn_cnn_arch(action_dim=A)).values()) + 257


def test_dqn_mlp_dueling_parameters():
    arch = archs.dqn_mlp((4,), 2, 128, 1, dueling=True)
    shapes = _pshapes(arch)
    assert shapes == [("dense/kernel", (4, 128)), ("dense/bias", (128,)), ("dense_1/kernel", (128, 2)), ("dense_1/bias", (2,)),
                      ("dense_2/kernel", (128, 1)), ("dense_2/bias", (1,))]
    assert sum(int(np.prod(s)) for _, s in shapes) == 1027
    assert arch["layers"][-1] == ("dueling", "dueling", ("dense_1", "dense_2"), {})
    assert _pshapes(orc.dqn_mlp_arch(dueling=True)) == shapes
    deep = archs.dqn_mlp((4,), 3, 64, 2, dueling=True)
    assert [l[0] for l in deep["layers"]] == ["dense", "dense_1", "dense_2", "dense_3", "dueling"]
    assert deep["layers"][-2][2] == "dense_1" and deep["layers"][-1][2] == ("dense_2", "dense_3")
    assert _pshapes(deep) == _pshapes(orc.dqn_mlp_arch((4,), 3, 64, 2, dueling=True))


def test_default_tables_unchanged():
    for A in (4, 18):
        assert archs.dqn_cnn((84, 84, 4), A) == archs.dqn_cnn((84, 84, 4), A, dueling=False)
        assert archs.dqn_cnn((84, 84, 4), A)["layers"] == orc.dqn_cnn_arch(action_dim=A)["layers"]
        assert orc.dqn_cnn_arch(action_dim=A, dueling=False) == archs.dqn_cnn((84, 84, 4), A)
    assert archs.dqn_mlp((4,), 2, 128, 1)["layers"] == orc.dqn_mlp_arch()["layers"]
    assert archs.dqn_mlp((4,), 2, 128, 1)["outputs"] == ["dense_1"]
    assert orc.dqn_mlp_arch(dueling=False) == archs.dqn_mlp((4,), 2, 128, 1)


@pytest.mark.parametrize("A", [2, 4, 9, 18])
def test_oracle_combine_matches_reference_golden(A):
    g = np.load(GOLDEN)
    value, adv, q = g["value_A%d" % A], g["adv_A%d" % A], g["q_A%d" % A]
    got = orc.dueling_combine(torch.from_numpy(value), torch.from_numpy(adv)).numpy()
    assert got.dtype == np.float32
    assert np.max(np.abs(got - q)) <= 1e-7 * np.max(np.abs(q))


def test_oracle_dueling_forward_through_mlp():
    arch = orc.dqn_mlp_arch(dueling=True)
    w = orc.init_weights(arch, seed=1)
    x = np.random.default_rng(0).standard_normal((6, 4)).astype(np.float32)
    t = orc.forward(arch, w, x, keep=True)
    np.testing.assert_array_equal(t["dueling"].numpy(), orc.dueling_combine(t["dense_1"], t["dense_2"]).numpy())
    assert t["dueling"].shape == (6, 2)


@pytest.mark.parametrize("A", [1, 3, 18])
def test_combine_gradient_closed_form(A):
    """float64 autograd of the combine: dvalue = g - mean(g), dadv = sum(g); for the TD step g = c e_a"""
    rng = np.random.default_rng(A)
    value = torch.from_numpy(rng.standard_normal((5, A))).requires_grad_(True)
    adv = torch.from_numpy(rng.standard_normal((5, 1))).requires_grad_(True)
    g = rng.standard_normal((5, A))
    dv, da = torch.autograd.grad((orc.dueling_combine(value, adv) * torch.from_numpy(g)).sum(), (value, adv))
    assert np.max(np.abs(dv.numpy() - (g - g.mean(1, keepdims=True)))) < 1e-12
    assert np.max(np.abs(da.numpy() - g.sum(1, keepdims=True))) < 1e-12
    a, c = A - 1, 0.37
    gt = np.zeros((1, A)); gt[0, a] = c
    dv, da = torch.autograd.grad((orc.dueling_combine(value[:1], adv[:1]) * torch.from_numpy(gt)).sum(), (value, adv))
    want = c * (np.eye(A)[a] - 1.0 / A)
    assert np.max(np.abs(dv.numpy()[0] - want)) < 1e-12 and abs(float(da[0, 0]) - c) < 1e-12
