"""PPO's DiagGaussian policy without a GPU: the Gaussian oracle against the reference's own DiagGaussianDist and PPO
losses (tests/golden/ppo_gauss.npz), its float64 gradients against the closed form the kernels use, the layer tables,
parameter names / shapes / counts, and the action types PPO accepts."""
import os

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from xingtian_b200.model import archs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ppo_gauss.npz")
PENDULUM = dict(state_dim=(3,), action_dim=1, hidden_sizes=(64, 64), activation="tanh", vf_share_layers=False)


def _close(got, want, tol=2e-5):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    err = float(np.max(np.abs(got - want)) / max(float(np.max(np.abs(want))), 1e-6))
    assert err <= tol, err


@pytest.mark.parametrize("A", [1, 3, 6])
def test_oracle_matches_reference_golden(A):
    g = {k[len("A%d_" % A):]: v for k, v in np.load(GOLDEN).items() if k.startswith("A%d_" % A)}
    clip, ent, vf_clip, cc = (float(x) for x in np.load(GOLDEN)["hyper"])
    t = lambda k: torch.from_numpy(g[k])   # noqa: E731
    mean, ls = t("mean"), t("log_std")
    x = orc.gauss_sample(mean, ls, t("normals"))
    _close(x, g["sample"])
    dls = orc.dist_log_std(mean, ls)
    _close(orc.gauss_log_prob(x, mean, dls), g["sample_logp"])
    _close(orc.gauss_neglog_prob(t("behav"), mean, dls), g["behav_neglogp"])
    _close(orc.gauss_entropy(dls), g["entropy"])
    loss = orc.ppo_gauss_loss(mean, ls, t("out_v"), t("behav"), t("old_logp"), t("adv"), t("old_v"), t("target_v"),
                              clip, ent, vf_clip, cc)
    _close(loss, g["total_loss"])
    # the fixture's inputs reach both sides of the surrogate clip and the clipped value loss
    ratio = np.exp(-g["behav_neglogp"] - g["old_logp"])
    assert (ratio < 1 - clip).any() and (ratio > 1 + clip).any()
    vc = g["old_v"] + np.clip(g["out_v"] - g["old_v"], -vf_clip, vf_clip)
    assert ((vc - g["target_v"]) ** 2 > (g["out_v"] - g["target_v"]) ** 2).any()


@pytest.mark.parametrize("A", [1, 3, 8])
def test_gradients_match_closed_form(A):
    """float64 autograd: dlogp/dmean = z/std, dlogp/dlog_std = z^2 - 1 (summed over the batch), dH/dlog_std = 1, and the
    entropy sends nothing into the mean (the * 0.0 branch)"""
    rng = np.random.default_rng(A)
    B = 7
    mean = torch.from_numpy(rng.standard_normal((B, A))).requires_grad_(True)
    ls = torch.from_numpy(rng.standard_normal((1, A)) * 0.5).requires_grad_(True)
    x = torch.from_numpy(rng.standard_normal((B, A)))
    dls = orc.dist_log_std(mean, ls)
    gm, gl = torch.autograd.grad(orc.gauss_log_prob(x, mean, dls).sum(), (mean, ls))
    std = np.exp(ls.detach().numpy())
    z = (x.numpy() - mean.detach().numpy()) / std
    assert np.max(np.abs(gm.numpy() - z / std)) < 1e-12
    assert np.max(np.abs(gl.numpy() - (z * z - 1).sum(0, keepdims=True))) < 1e-12
    gm, gl = torch.autograd.grad(orc.gauss_entropy(orc.dist_log_std(mean, ls)).mean(), (mean, ls))
    assert np.max(np.abs(gm.numpy())) == 0.0 and np.max(np.abs(gl.numpy() - 1.0)) < 1e-12


def test_gaussian_tables_and_names():
    cat = archs.ppo_mlp(**PENDULUM)
    gauss = archs.ppo_mlp(**PENDULUM, diag_gaussian=True)
    assert gauss["layers"][:-1] == cat["layers"] and gauss["outputs"] == cat["outputs"]
    assert gauss["layers"][-1] == ("pi_logstd", "logstd", None, dict(n=1))
    shapes = orc.param_shapes(gauss)
    assert list(shapes)[-1] == "pi_logstd" and shapes["pi_logstd"] == (1, 1)
    assert list(shapes)[:-1] == list(orc.param_shapes(orc.ppo_mlp_arch((3,), 1))) == list(orc.param_shapes(cat))
    assert sum(int(np.prod(s)) for s in shapes.values()) == 2 * (3 * 64 + 64 + 64 * 64 + 64) + 65 + 65 + 1 == 8963
    assert gauss["layers"] == orc.ppo_mlp_arch(state_dim=(3,), action_dim=1, diag_gaussian=True)["layers"]
    cnn = archs.ppo_cnn((84, 84, 4), 3, [512], "relu", True, diag_gaussian=True)
    assert cnn["layers"][-1] == ("pi_logstd", "logstd", None, dict(n=3))
    assert cnn["layers"] == orc.ppo_cnn_arch(action_dim=3, hidden_sizes=(512,), diag_gaussian=True)["layers"]
    assert orc.param_shapes(cnn)["pi_logstd"] == (1, 3)
    w = orc.init_weights(gauss, seed=0)
    assert list(w) == list(shapes) and not w["pi_logstd"].any()


def test_categorical_tables_unchanged():
    for kw in (PENDULUM, dict(PENDULUM, state_dim=(4,), action_dim=2)):
        assert archs.ppo_mlp(**kw) == archs.ppo_mlp(**kw, diag_gaussian=False)
        assert archs.ppo_mlp(**kw)["layers"] == orc.ppo_mlp_arch(kw["state_dim"], kw["action_dim"])["layers"]
    for A in (4, 18):
        a = archs.ppo_cnn((84, 84, 4), A, [256], "relu", True)
        assert a == archs.ppo_cnn((84, 84, 4), A, [256], "relu", True, diag_gaussian=False)
        assert a["layers"] == orc.ppo_cnn_arch(action_dim=A)["layers"]


@pytest.mark.parametrize("model", ["PpoMlp", "PpoCnn"])
@pytest.mark.parametrize("action_type", ["MultiCategorical", "Beta"])
def test_other_action_types_raise(model, action_type):
    import xingtian_b200  # noqa: F401  (registers the models)
    from xingtian_b200.registry import Registers
    info = {"state_dim": [3] if model == "PpoMlp" else [84, 84, 4], "action_dim": 2,
            "model_config": {"action_type": action_type}}
    with pytest.raises(NotImplementedError, match="action type: {} not match any implemented distributions.".format(action_type)):
        Registers.model[model](info)
