"""IMPALA with the Keras learner, host side (no GPU): the oracle against the reference's own code (golden fixture), the
loss gradient against finite differences, the plugins' registry keys and layer tables, the host shuffle order and the
trajectory validation."""
import os

import numpy as np
import pytest
import torch

import impala_keras_oracle as iko
from oracle import xt_oracle as orc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "impala_keras.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_vtrace_matches_reference(gold, case):
    """_train_proc: pg_adv and target value of every training row, the slices handed to actor.train (state ids skip the
    bootstrap state of each trajectory) and the mean of the slice losses"""
    g = {k[3:]: gold[k] for k in gold.files if k.startswith("c%d_" % case)}
    n, L, A, batch = (int(x) for x in g["cfg"])
    pg, tv = iko.vtrace(g["probs"].reshape(n, L + 1, A), g["values"].reshape(n, L + 1), g["behav"].reshape(n, L, A),
                        g["amat"].reshape(n, L, A), g["reward"].reshape(n, L), g["done"].reshape(n, L))
    np.testing.assert_allclose(pg, g["pg_adv"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(tv, g["tv"], rtol=0, atol=1e-12)
    rows = np.arange(n * L)
    np.testing.assert_array_equal(g["state_ids"], rows + rows // L)
    np.testing.assert_array_equal(g["slice_amat"], g["amat"])
    sizes = [min(batch, n * L - s) for s in range(0, n * L, batch)]
    np.testing.assert_array_equal(g["slice_sizes"], sizes)
    assert float(g["mean_loss"]) == np.mean(np.arange(1, len(sizes) + 1))


@pytest.mark.parametrize("case", [0, 1, 2])
def test_loss_matches_reference(gold, case):
    """impala_loss of both models: the MLP's scalar and the CNN's per-row vector (whose batch mean Keras takes)"""
    pre = "loss%d_" % case
    p, y, adv = gold[pre + "probs"], gold[pre + "y"], gold[pre + "adv"]
    want = iko.impala_loss_value(p, y, adv)
    assert abs(want - float(gold[pre + "mlp"])) < 1e-7 * max(1.0, abs(want))
    assert abs(want - float(np.mean(gold[pre + "cnn"], dtype=np.float64))) < 1e-7 * max(1.0, abs(want))
    # the per-row loss of the oracle with a zero value term is the CNN closure's per-row vector
    logits = torch.from_numpy(np.log(p.astype(np.float64)))
    rl = iko.row_losses(logits, torch.zeros(len(p), dtype=torch.float64), torch.from_numpy(y.astype(np.float64)),
                        torch.from_numpy(adv.astype(np.float64)), torch.zeros(len(p), dtype=torch.float64))
    np.testing.assert_allclose(rl.numpy(), gold[pre + "cnn"], rtol=1e-6, atol=1e-7)


def test_loss_gradient_matches_finite_differences():
    rng = np.random.default_rng(3)
    B, A = 6, 5
    logits = torch.from_numpy(rng.standard_normal((B, A)) * 2).requires_grad_(True)
    v = torch.from_numpy(rng.standard_normal(B)).requires_grad_(True)
    y = torch.from_numpy(np.eye(A)[rng.integers(0, A, B)])
    adv, tv = torch.from_numpy(rng.standard_normal(B)), torch.from_numpy(rng.standard_normal(B))
    f = lambda lg, vv: float(iko.row_losses(lg, vv, y, adv, tv).mean())   # noqa: E731
    gl, gv = torch.autograd.grad(iko.row_losses(logits, v, y, adv, tv).mean(), (logits, v))
    h = 1e-6
    lg0, v0 = logits.detach(), v.detach()
    for b in range(B):
        for i in range(A):
            e = torch.zeros_like(lg0); e[b, i] = h
            assert abs((f(lg0 + e, v0) - f(lg0 - e, v0)) / (2 * h) - float(gl[b, i])) < 1e-8
        e = torch.zeros_like(v0); e[b] = h
        assert abs((f(lg0, v0 + e) - f(lg0, v0 - e)) / (2 * h) - float(gv[b])) < 1e-8
    # the closed form the device kernel evaluates: dz_j = p_j (g_j - sum_i p_i g_i) / (A B), dv = (v - tv) / B
    p = torch.softmax(lg0, -1)
    g = -adv[:, None] * y / (p + 1e-10) + 0.01 * (torch.log(p + 1e-10) + p / (p + 1e-10))
    dz = p * (g - (p * g).sum(-1, keepdim=True)) / (A * B)
    np.testing.assert_allclose(dz.numpy(), gl.numpy(), rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(((v0 - tv) / B).numpy(), gv.numpy(), rtol=1e-12)


def test_keras_adam_decay_closed_form():
    p = [torch.zeros(3, dtype=torch.float64)]
    with orc.precision("f64"):
        opt = iko.KerasAdam(p, 0.01, decay=0.5)
        for it in range(3):
            opt.step([torch.ones(3, dtype=torch.float64)])
            assert opt.lr == pytest.approx(0.01 / (1 + 0.5 * it))
    # constant gradient: m_hat / sqrt(v_hat) = 1, so every step moves by its decayed lr (up to the epsilon term)
    assert float(p[0][0]) == pytest.approx(-sum(0.01 / (1 + 0.5 * i) for i in range(3)), rel=1e-5)


def test_registry_and_layer_tables():
    from xingtian_b200.registry import Registers
    from xingtian_b200.model import archs
    assert "IMPALA" in Registers.algorithm and "ImpalaMlp" in Registers.model and "ImpalaCnn" in Registers.model
    for mine, ref, count in ((archs.impala_mlp((4,), 2, 128, 1), iko.impala_mlp_arch(), 1027),
                             (archs.impala_keras_cnn((84, 84, 4), 4), iko.impala_cnn_arch(), 882341)):
        assert mine == ref
        shapes = orc.param_shapes(mine)
        assert sum(int(np.prod(s)) for s in shapes.values()) == count
        assert list(shapes)[-4:] == ["output_actions/kernel", "output_actions/bias", "output_value/kernel", "output_value/bias"]
    assert list(orc.param_shapes(archs.impala_mlp((4,), 3, 64, 2))) == [
        "dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias", "output_actions/kernel", "output_actions/bias",
        "output_value/kernel", "output_value/bias"]
    # ImpalaCnnOpt's module globals are not those of the new models
    from xingtian_b200.model import impala, impala_cnn, impala_mlp
    assert impala.__dict__ is not impala_cnn.__dict__ and impala_mlp.__dict__ is not impala_cnn.__dict__


def test_shuffle_order_follows_reference_call_sequence():
    """one np.random.shuffle(np.arange(len)) per BATCH_SIZE slice, in order, the slice offset added"""
    from xingtian_b200.algorithm.impala import slice_orders
    from xingtian_b200.model.impala_keras import fit_order
    np.random.seed(7)
    got = slice_orders(1000, 400)
    np.random.seed(7)
    want = []
    for s, n in ((0, 400), (400, 400), (800, 200)):
        idx = np.arange(n)
        np.random.shuffle(idx)
        want.append(idx + s)
    np.testing.assert_array_equal(got, np.concatenate(want))
    np.random.seed(8)
    o = fit_order(300)
    np.random.seed(8)
    batches = iko.fit_batches(300)
    assert [len(b) for b in batches] == [128, 128, 44]
    np.testing.assert_array_equal(o, np.concatenate(batches))


def test_trajectory_validation():
    """prepare_data rejects trajectories that do not match episode_len before touching the device"""
    from xingtian_b200.algorithm.impala import IMPALA
    alg = object.__new__(IMPALA)
    alg.episode_len = 5
    alg.actor = type("A", (), {"action_dim": 3})()
    ok = dict(cur_state=np.zeros((6, 4)), real_action=np.eye(3)[[0, 1, 2, 0, 1]], action=np.full((5, 3), 1 / 3),
              reward=[0.0] * 5, done=[False] * 5)
    s, a, d, p, r = alg._data_proc(ok)
    assert s.shape == (6, 4) and a.dtype == np.float32 and d.dtype == np.bool_ and r.shape == (5,)
    for key, bad in (("cur_state", np.zeros((5, 4))), ("real_action", np.eye(3)[[0, 1, 2, 0]]), ("action", np.ones((5, 2))),
                     ("reward", [0.0] * 6), ("done", [False] * 4)):
        with pytest.raises(ValueError):
            alg._data_proc(dict(ok, **{key: bad}))
