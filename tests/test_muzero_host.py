"""MuZero on the host: the support transforms, the layer tables, their parameter counts and weight-list order, and the
float64 oracle's gradient against finite differences."""
import numpy as np
import pytest
import torch

import muzero_oracle as mo
from xingtian_b200.model import archs


def test_support_sizes():
    # muzero_model.py:47-52 for the two Atari configs and the defaults
    assert (mo.support_size(0, 500), mo.support_size(0, 50)) == (23, 8)       # muzero_breakout.yaml
    assert (mo.support_size(-21, 21), mo.support_size(-2, 2)) == (7, 3)       # muzero_pong.yaml
    assert (mo.support_size(0, 60000), mo.support_size(-300, 300)) == (305, 26)


def test_value_transform_round_trip():
    x = np.linspace(-500.0, 60000.0, 997)
    np.testing.assert_allclose(mo.h_inv(mo.h(x)), x, rtol=1e-9, atol=1e-6)
    # the expectation of a two-hot row recovers the clipped scalar
    for vmin, vmax in ((0, 500), (-21, 21), (0, 60000)):
        S = mo.support_size(vmin, vmax)
        xs = np.random.default_rng(0).uniform(vmin - 5, vmax + 5, 64)
        t = mo.two_hot(xs, S, vmin, vmax)
        np.testing.assert_allclose(t.sum(-1), 1.0, atol=1e-12)
        np.testing.assert_allclose(mo.support_value(t, vmin, vmax), np.clip(xs, vmin, vmax), rtol=1e-9, atol=1e-6)


def test_tables_param_counts_and_list_order():
    # counted by hand from the reference's layers (muzero_cnn.py:42-67, muzero_mlp.py:41-63)
    br = archs.muzero_cnn((84, 84, 4), 4, 23, 8)
    assert [mo.param_count(a) for a in br] == [846208, 133768, 36379]
    assert sum(mo.param_count(a) for a in br) == 1016355
    assert sum(mo.param_count(a) for a in archs.muzero_cnn((84, 84, 4), 6, 7, 3)) == 1014416
    assert sum(mo.param_count(a) for a in archs.muzero_mlp((4,), 2, 305, 26)) == 23253
    # Keras weight list: representation, dynamics, prediction; within the prediction model out_p precedes out_v, the
    # order of Keras's _map_graph_network walk from outputs [out_p, out_v] (derived from its rules, not run under TF)
    rep, dyn, pred = br
    assert [l[0] for l in dyn["layers"]] == ["dense", "dense_1", "out_h", "out_r"]
    assert [l[0] for l in pred["layers"]] == ["dense", "out_p", "out_v"]
    shapes = sum((mo.weight_shapes(a) for a in br), [])
    assert shapes[:2] == [(8, 8, 4, 32), (32,)] and shapes[6:8] == [(3136, 256), (256,)]
    assert shapes[8] == (260, 256) and shapes[-4:] == [(128, 4), (4,), (128, 23), (23,)]


def _mlp_setup(seed, B=3, K=5, A=2, vrange=(0, 20), rrange=(-2, 2)):
    Sv, Sr = mo.support_size(*vrange), mo.support_size(*rrange)
    ar = archs.muzero_mlp((4,), A, Sv, Sr, hidden1=8, hidden2=4)
    rng = np.random.default_rng(seed)
    weights = [rng.normal(0, 0.5, s) for s in sum((mo.weight_shapes(a) for a in ar), [])]
    obs = rng.normal(size=(B, 4))
    action = rng.integers(0, A, (B, K))
    tv = rng.uniform(vrange[0], vrange[1], (B, K + 1))
    tr = rng.uniform(rrange[0], rrange[1], (B, K + 1))
    tp = rng.dirichlet(np.ones(A), (B, K + 1))
    return ar, weights, obs, action, tv, tr, tp, K, vrange, rrange


def test_oracle_gradient_matches_finite_differences_without_scaling_rules():
    """With the 1/K and 0.5 rules the autograd gradient is not the derivative of the loss value; with K = 1 the 0.5
    rule has no effect (no dynamics step follows) and the 1/K rule is the identity, so the gradient must match finite differences."""
    ar, w, obs, action, tv, tr, tp, _, vr, rr = _mlp_setup(1, B=2, K=1)
    params = [torch.tensor(x, requires_grad=True) for x in w]
    loss = mo.train_loss(ar, params, obs, action, tv, tr, tp, 1, vr, rr)
    loss.backward()
    rng = np.random.default_rng(2)
    for pi in rng.choice(len(w), 6, replace=False):
        idx = tuple(rng.integers(0, s) for s in w[pi].shape)
        eps = 1e-6
        vals = []
        for sgn in (1, -1):
            p2 = [torch.tensor(x) for x in w]
            p2[pi][idx] += sgn * eps
            vals.append(float(mo.train_loss(ar, p2, obs, action, tv, tr, tp, 1, vr, rr)))
        fd = (vals[0] - vals[1]) / (2 * eps)
        assert abs(fd - float(params[pi].grad[idx])) < 1e-6 * max(1.0, abs(fd)), (pi, idx)


def test_oracle_loss_value_is_unscaled():
    """scale_gradient changes gradients only: the oracle's loss value is the plain sum of the cross-entropy terms."""
    ar, w, obs, action, tv, tr, tp, K, vr, rr = _mlp_setup(3, K=3)
    with torch.no_grad():
        p2 = [torch.tensor(x) for x in w]
        val = float(mo.train_loss(ar, p2, obs, action, tv, tr, tp, K, vr, rr))
    rep_a, dyn_a, pred_a = ar
    rep_w, dyn_w, pred_w = mo.split(ar, [torch.tensor(x) for x in w])
    Sv, Sr = pred_a["layers"][-1][3]["n"], dyn_a["layers"][-1][3]["n"]
    tv2, tr2 = torch.from_numpy(mo.two_hot(tv, Sv, *vr)), torch.from_numpy(mo.two_hot(tr, Sr, *rr))
    tpt = torch.as_tensor(tp)
    hid = mo.forward(rep_a, rep_w, torch.as_tensor(obs))["dense_1"]
    po = mo.forward(pred_a, pred_w, hid)
    total = mo.cross_entropy(po["out_p"], tpt[:, 0]) + mo.cross_entropy(po["out_v"], tv2[:, 0])
    for i in range(K):
        x = torch.cat([hid, torch.nn.functional.one_hot(torch.as_tensor(action[:, i]), 2).double()], -1)
        do = mo.forward(dyn_a, dyn_w, x)
        hid = do["out_h"]
        po = mo.forward(pred_a, pred_w, hid)
        total = total + mo.cross_entropy(do["out_r"], tr2[:, i]) + mo.cross_entropy(po["out_p"], tpt[:, i + 1]) + \
            mo.cross_entropy(po["out_v"], tv2[:, i + 1])
    assert abs(float(total) - val) < 1e-12 * max(1.0, abs(val))


def test_unknown_obs_type_rejected_before_cuda():
    from xingtian_b200.model.muzero import MuzeroModel
    with pytest.raises(ValueError):
        MuzeroModel.__init__(object.__new__(MuzeroModel), {"state_dim": [84, 84, 4], "action_dim": 6,
                                                           "model_config": {"obs_type": "float16"}})
