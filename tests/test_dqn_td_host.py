"""The float64 DQN TD step of the oracle, the yardstick of tests/test_gpu_dqn_td.py, on the CPU: under precision("f64")
dqn_targets is the per-row target loop of DQN.train in float64 (double DQN taking the first maximum of the online row, as
dqn_td_target does), and the autograd gradients of DqnLearner's loss are the closed forms dqn_loss_kernel and
DuelingTdLoss implement; the default precision still returns float32."""
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc


def _naive_targets(y_online, tq, act, rew, done, gamma, qo=None, disc=None):
    """y = y_online with y[k, a_k] = r_k, or r_k + g_k Q_target(s'_k, a*) unless done; a* = argmax of the target row, or
    of the online row for double DQN (first maximum); g_k = disc[k] when given, else gamma.  One row at a time."""
    y = np.array(y_online, np.float64)
    for k in range(len(y)):
        row = qo[k] if qo is not None else tq[k]
        best = 0
        for i in range(1, len(row)):
            if row[i] > row[best]:
                best = i
        g = float(disc[k]) if disc is not None else gamma
        y[k, act[k]] = float(rew[k]) if done[k] else float(rew[k]) + g * float(tq[k][best])
    return y


def _td_inputs(B, A, seed):
    rng = np.random.default_rng(seed)
    y0 = rng.standard_normal((B, A)).astype(np.float32)
    tq = rng.standard_normal((B, A)).astype(np.float32)
    qo = rng.standard_normal((B, A)).astype(np.float32)
    # ties in the online rows: the maximum repeated at a later action whose target value differs
    for k in range(0, B, 3):
        i, j = sorted(rng.choice(A, 2, replace=False))
        qo[k, i] = qo[k, j] = qo[k].max() + 1.0
        tq[k, j] = tq[k, i] + 0.5
    act = rng.integers(0, A, B).astype(np.int32)
    rew = (3 * rng.standard_normal(B)).astype(np.float32)
    done = rng.random(B) < 0.25
    done[0], done[1] = True, False
    disc = np.where(done, 0.0, np.float32(0.99) ** rng.integers(1, 4, B)).astype(np.float32)
    disc[2::5] = 0.0                       # a window that hit a terminal step, on rows that are not done
    return y0, tq, qo, act, rew, done, disc


@pytest.mark.parametrize("B,A,gamma", [(2, 2, 0.99), (37, 4, 0.99), (64, 18, 1.0), (50, 6, 0.0)])
@pytest.mark.parametrize("form", ["plain", "double", "disc", "double_disc"])
def test_float64_targets_are_the_naive_loop(B, A, gamma, form):
    y0, tq, qo, act, rew, done, disc = _td_inputs(B, A, B * 10 + A)
    qo_, disc_ = (qo if "double" in form else None), (disc if "disc" in form else None)
    g = float(np.float32(gamma))
    with orc.precision("f64"):
        y = orc.dqn_targets(y0, tq, act, rew, done, g, qo_, disc_)
    assert y.dtype == np.float64
    want = _naive_targets(y0, tq, act, rew, done, g, qo_, disc_)
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    # the regimes occur: done rows, disc 0 on rows that are not done, tied online maxima whose target values differ
    assert done.any() and not done.all()
    if "disc" in form and B > 2:
        assert ((disc == 0) & ~done).any()
    if "double" in form:
        tied = [k for k in range(B) if (qo[k] == qo[k].max()).sum() > 1]
        assert tied
        last = [A - 1 - int(np.argmax(qo[k][::-1])) for k in tied]
        assert any(tq[k, np.argmax(qo[k])] != tq[k, j] for k, j in zip(tied, last))
    # the default precision keeps the reference's float32 y
    assert orc.dqn_targets(y0, tq, act, rew, done, g, qo_, disc_).dtype == np.float32


def _identity_arch(B, A, dueling):
    """obs = the B x B identity: Q row b is the kernel's row b (+ bias), so d loss / d kernel row b is d loss / d Q row b"""
    if dueling:
        layers = [("value", "dense", "obs", dict(n=A, act=None)), ("adv", "dense", "obs", dict(n=1, act=None)),
                  ("q", "dueling", ("value", "adv"), {})]
    else:
        layers = [("q", "dense", "obs", dict(n=A, act=None))]
    return dict(input_dtype="float32", state_dim=(B,), scale=1.0, layers=layers, outputs=["q"])


def _learner(B, A, dueling, seed, double=False):
    rng = np.random.default_rng(seed)
    arch = _identity_arch(B, A, dueling)
    w = OrderedDict((k, rng.standard_normal(s).astype(np.float32)) for k, s in orc.param_shapes(arch).items())
    wt = OrderedDict((k, rng.standard_normal(s).astype(np.float32)) for k, s in orc.param_shapes(arch).items())
    return arch, w, wt, orc.DqnLearner(arch, w, double_dqn=double, target_weights=wt)


@pytest.mark.parametrize("B,A", [(1, 1), (7, 4), (33, 6)])
@pytest.mark.parametrize("dueling", [False, True])
@pytest.mark.parametrize("huber", [0.0, 1.0])
def test_float64_loss_gradients_are_the_kernel_closed_forms(B, A, dueling, huber):
    """dq = c e_a with c = 2 w diff / (B A) (squared error) or w clamp(diff, -delta, delta) / (B A) (Huber, on both
    sides of delta and at |diff| = delta); dueling: dvalue = c (e_a - 1 / A), dadv = c.  The loss is
    1/(B A) sum_b w_b e_b, and td_abs = |diff|"""
    rng = np.random.default_rng(B * 100 + A)
    with orc.precision("f64"):
        arch, w, wt, ln = _learner(B, A, dueling, B + A, double=True)
        eye = np.eye(B, dtype=np.float32)
        act = rng.integers(0, A, B).astype(np.int32)
        done = rng.random(B) < 0.5
        rew = (3 * rng.standard_normal(B)).astype(np.float32)
        weights = rng.uniform(0.0, 2.0, B).astype(np.float32)
        weights[0] = 0.0
        disc = rng.uniform(0.5, 1.0, B).astype(np.float32)
        if huber:
            # done rows: y = r exactly; move Q(s, a) to chosen TD errors, |diff| = delta exactly among them
            done[:] = True
            offs = np.resize([-2.5, -1.0, -0.25, 0.5, 1.0, 3.0], B)
            q = ln.predict(eye)
            shift = rew.astype(np.float64) + offs - q[np.arange(B), act]
            kname = "q/kernel" if not dueling else "adv/kernel"
            # adv (1 wide) adds to every action alike; without dueling move the taken entry of the kernel row
            p = ln.named()[kname]
            with torch.no_grad():
                if dueling:
                    p[np.arange(B), 0] += torch.from_numpy(shift)
                else:
                    p[np.arange(B), torch.from_numpy(act.astype(np.int64))] += torch.from_numpy(shift)
        loss, grads, y, td_abs = ln.loss_and_grads(eye, act, rew, eye, done, disc=disc, huber=huber, weights=weights)
        assert loss.dtype == torch.float64 and y.dtype == np.float64
        g = dict(zip(ln.names, (t.numpy() for t in grads)))
        q = ln.predict(eye)
    diff = q[np.arange(B), act] - y[np.arange(B), act]
    if huber:
        np.testing.assert_allclose(diff, offs, rtol=0, atol=1e-12)
        c = weights * np.clip(diff, -huber, huber) / (B * A)
        per = np.where(np.abs(diff) <= huber, 0.5 * diff * diff, huber * (np.abs(diff) - 0.5 * huber))
    else:
        c = 2.0 * weights * diff / (B * A)
        per = diff * diff
    np.testing.assert_allclose(float(loss.detach()), float((weights * per).sum() / (B * A)), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(td_abs, np.abs(diff), rtol=1e-12, atol=1e-14)
    e_a = np.eye(A)[act]
    if dueling:
        np.testing.assert_allclose(g["value/kernel"], c[:, None] * (e_a - 1.0 / A), rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(g["adv/kernel"][:, 0], c, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(g["value/bias"], (c[:, None] * (e_a - 1.0 / A)).sum(0), rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(g["adv/bias"], [c.sum()], rtol=1e-12, atol=1e-14)
    else:
        np.testing.assert_allclose(g["q/kernel"], c[:, None] * e_a, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(g["q/bias"], (c[:, None] * e_a).sum(0), rtol=1e-12, atol=1e-14)


def test_target_weights_and_unweighted_results():
    """the target net takes its own weights (double DQN then differs from plain DQN); weights=None is the unweighted
    loss, and the fp32 learner still builds the float32 y of the reference"""
    B, A = 9, 4
    arch, w, wt, ln = _learner(B, A, False, 3)
    eye = np.eye(B, dtype=np.float32)
    np.testing.assert_array_equal(ln.predict(eye, target=True), wt["q/kernel"] + wt["q/bias"])
    np.testing.assert_array_equal(ln.predict(eye), w["q/kernel"] + w["q/bias"])
    rng = np.random.default_rng(0)
    act, rew, done = rng.integers(0, A, B), rng.standard_normal(B).astype(np.float32), np.zeros(B, bool)
    l0, g0, y0, _ = ln.loss_and_grads(eye, act, rew, eye, done)
    l1, g1, y1, _ = ln.loss_and_grads(eye, act, rew, eye, done, weights=np.ones(B, np.float32))
    assert y0.dtype == np.float32 and float(l0) == float(l1)
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)
    dbl = orc.DqnLearner(arch, w, double_dqn=True, target_weights=wt)
    assert not np.array_equal(dbl.loss_and_grads(eye, act, rew, eye, done)[2], y0)
    same = orc.DqnLearner(arch, w)
    np.testing.assert_array_equal(same.predict(eye, target=True), same.predict(eye))
