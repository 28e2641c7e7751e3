"""The hidden activations of PPO's ACTIVATION_MAP without a GPU: the torch and numpy float64 restatements against each
other, the closed forms and the reference's own gelu (tests/golden/activations.npz), the derivative rules the kernels
use against autograd, the name tables against the fixture and include/xtb200.h, and the model-config surface."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import np_f64
from oracle import xt_oracle as orc
from xingtian_b200 import capi
from xingtian_b200.model import archs

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "activations.npz")
HEADER = os.path.join(HERE, "..", "include", "xtb200.h")


def _grid():
    x = np.concatenate([np.linspace(-30, 30, 6001), np.linspace(-1e-3, 1e-3, 201), [1e-12, -1e-12, 1e-300, -1e-300]])
    return np.unique(x)


@pytest.mark.parametrize("act", np_f64.NEW)
def test_torch_and_numpy_f64_agree(act):
    x = _grid()
    t = orc._ACT[act](torch.from_numpy(x)).numpy()
    n = np_f64._ACT[act](x)
    assert t.dtype == np.float64 and n.dtype == np.float64
    # relative 1e-13; gelu's 1 + tanh(.) cancels for x << 0, where one double ulp of it, times |x|, is what is left
    bound = 1e-13 * np.abs(n) + np.finfo(np.float64).eps * np.abs(x)
    assert np.all(np.abs(t - n) <= bound), float(np.max(np.abs(t - n) / (bound + 1e-300)))


def test_closed_forms_and_constants():
    x = _grid()
    f = {k: np_f64._ACT[k](x) for k in np_f64.NEW}
    with np.errstate(over="ignore"):
        np.testing.assert_allclose(f["sigmoid"], 1 / (1 + np.exp(-x)), rtol=1e-15)
    np.testing.assert_allclose(f["softplus"], np.logaddexp(0.0, x), rtol=1e-15)          # log(1 + e^x), accurately
    np.testing.assert_allclose(f["softsign"], x / (1 + np.abs(x)), rtol=1e-15)
    np.testing.assert_array_equal(f["leaky_relu"], np.maximum(x, 0.2 * x))
    np.testing.assert_allclose(f["elu"], np.where(x > 0, x, np.exp(np.minimum(x, 0)) - 1), rtol=1e-9, atol=1e-15)
    assert np_f64.SELU_SCALE == 1.0507009873554805 and np_f64.SELU_ALPHA == 1.6732632423543772
    np.testing.assert_allclose(f["selu"][x < 0] / np_f64.SELU_SCALE / np_f64.SELU_ALPHA, np.expm1(x[x < 0]), rtol=1e-15)
    np.testing.assert_allclose(f["swish"], x / (1 + np.exp(-x)), rtol=1e-14)
    np.testing.assert_allclose(f["gelu"], 0.5 * x * (1 + np.tanh(np.sqrt(2 / np.pi) * (x + 0.044715 * x ** 3))), rtol=1e-15)
    assert abs(f["softplus"][np.searchsorted(x, 30.0)] - 30.0) < 1e-12          # stable at large x
    assert f["softplus"][0] > 0                                                  # and at large negative x


def test_gelu_matches_reference_golden():
    g = np.load(GOLDEN)
    x = g["x"].astype(np.float64)
    ref = g["gelu"].astype(np.float64)
    ours = orc._ACT["gelu"](torch.from_numpy(x)).numpy()
    # float32 rounding of the reference's eager float32 ops: a few ulp of the largest intermediate
    tol = 4 * np.finfo(np.float32).eps * np.maximum(np.abs(x), np.abs(ref)) + 1e-30
    assert np.all(np.abs(ours - ref) <= tol), float(np.max(np.abs(ours - ref) / tol))
    with orc.precision("f32"):
        got32 = orc._ACT["gelu"](torch.from_numpy(g["x"])).numpy()
    assert got32.dtype == np.float32
    assert np.all(np.abs(got32 - ref) <= tol)


@pytest.mark.parametrize("act", np_f64.NEW)
def test_kernel_derivative_rules_match_autograd(act):
    x = _grid()
    if act in ("leaky_relu", "selu", "elu", "softplus"):
        # away from the kink at 0 (softplus has none, but autograd takes the subgradients of max(x, 0) and |x| there)
        x = x[np.abs(x) > 1e-9]
    z = torch.from_numpy(x).requires_grad_(True)
    y = orc._ACT[act](z)
    (g,) = torch.autograd.grad(y.sum(), z)
    rule = np_f64.grad_rule(act, y.detach().numpy(), x)
    g = g.numpy()
    err = np.abs(rule - g) / np.maximum(np.abs(g), 1.0)
    assert float(np.max(err)) <= 1e-10, (act, float(np.max(err)), x[np.argmax(err)])


def test_act_table_matches_reference_map_and_header():
    keys = set(str(k) for k in np.load(GOLDEN)["act_map_keys"])
    assert len(keys) == 10
    assert set(capi.ACT) == keys | {"linear", None}
    with open(HEADER) as f:
        src = f.read()
    body = re.search(r"enum xtb_act \{([^}]*)\}", src).group(1)
    enum = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r"XTB_ACT_(\w+)\s*=\s*(\d+)", body)}
    want = dict(enum)
    want["linear"] = want.pop("none")
    assert {k: v for k, v in capi.ACT.items() if k is not None} == want
    assert capi.ACT[None] == 0
    assert sorted(enum.values()) == list(range(11))


@pytest.mark.parametrize("model", ["PpoMlp", "PpoCnn"])
def test_unknown_activation_raises_reference_keyerror(model):
    import xingtian_b200  # noqa: F401  (registers the models)
    from xingtian_b200.registry import Registers
    info = {"state_dim": [3] if model == "PpoMlp" else [84, 84, 4], "action_dim": 2, "model_config": {"activation": "mish"}}
    with pytest.raises(KeyError, match="activation mish not implemented."):
        Registers.model[model](info)


@pytest.mark.parametrize("act", sorted(k for k in capi.ACT if k is not None))
def test_archs_equal_oracle_tables(act):
    for A, share in ((4, True), (18, False)):
        assert archs.ppo_cnn((84, 84, 4), A, [256], act, share)["layers"] == orc.ppo_cnn_arch(
            action_dim=A, activation=act, vf_share_layers=share)["layers"]
    for sd, A in (((4,), 2), ((3,), 1)):
        assert archs.ppo_mlp(sd, A, [64, 64], act, False)["layers"] == orc.ppo_mlp_arch(
            sd, A, activation=act)["layers"]
