"""CPU tier: the float64 QMIX restatement (tests/qmix_oracle.py) that the device training step is checked against."""
import math

import numpy as np
import torch

from oracle import xt_oracle as orc
import qmix_oracle as qo


def _weights(rng, obs_dim, H, A, n, E, he, sd):
    w = {}
    shapes = [("dense/kernel", (obs_dim, H)), ("dense/bias", (H,)), (qo.GATES_K, (2 * H, 2 * H)), (qo.GATES_B, (2 * H,)),
              (qo.CAND_K, (2 * H, H)), (qo.CAND_B, (H,)), ("dense_1/kernel", (H, A)), ("dense_1/bias", (A,))]
    widths = dict(zip(qo.MIX_LAYERS, (he, E * n, E, he, E, E, 1)))
    srcs = dict(zip(qo.MIX_LAYERS, (sd, he, sd, sd, he, sd, E)))
    for name in qo.MIX_LAYERS:
        shapes += [(name + "/kernel", (srcs[name], widths[name])), (name + "/bias", (widths[name],))]
    for name, s in shapes:
        w[name] = rng.normal(scale=0.4, size=s)
    return w


def test_gru_cell_matches_scalar_loop():
    rng = np.random.default_rng(0)
    H, X = 3, 3
    w = {qo.GATES_K: rng.normal(size=(X + H, 2 * H)), qo.GATES_B: rng.normal(size=2 * H),
         qo.CAND_K: rng.normal(size=(X + H, H)), qo.CAND_B: rng.normal(size=H)}
    x, h = rng.normal(size=X), rng.normal(size=H)
    sig = lambda z: 1 / (1 + math.exp(-z))
    xh = list(x) + list(h)
    g = [sig(sum(xh[k] * w[qo.GATES_K][k, j] for k in range(X + H)) + w[qo.GATES_B][j]) for j in range(2 * H)]
    r, u = g[:H], g[H:]
    xrh = list(x) + [r[k] * h[k] for k in range(H)]
    c = [math.tanh(sum(xrh[k] * w[qo.CAND_K][k, j] for k in range(X + H)) + w[qo.CAND_B][j]) for j in range(H)]
    want = [u[j] * h[j] + (1 - u[j]) * c[j] for j in range(H)]
    with orc.precision("f64"):
        got = qo.gru_cell(qo._t(x)[None], qo._t(h)[None], {k: qo._t(v) for k, v in w.items()})[0].numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_outputs_past_the_sequence_length_are_zero():
    rng = np.random.default_rng(1)
    w = _weights(rng, 5, 4, 3, 2, 4, 6, 7)
    with orc.precision("f64"):
        wt = {k: qo._t(v) for k, v in w.items()}
        obs = qo._t(rng.normal(size=(2, 6, 2, 5)))
        h0 = qo._t(rng.normal(size=(4, 4)))
        q, hT = qo.agent_forward(wt, obs, [4, 4, 2, 0], h0)     # sequence b n + a: episode 1's agent 1 has length 0
        q, hT, h0 = q.numpy(), hT.numpy(), h0.numpy()
    bias = w["dense_1/bias"]
    np.testing.assert_allclose(q[0, 4:], np.broadcast_to(bias, q[0, 4:].shape), rtol=0, atol=0)
    np.testing.assert_allclose(q[1, 2:], np.broadcast_to(bias, q[1, 2:].shape), rtol=0, atol=0)
    np.testing.assert_allclose(q[1, :, 1], np.broadcast_to(bias, q[1, :, 1].shape), rtol=0, atol=0)
    assert np.abs(q[0, :4] - bias).max() > 1e-3 and np.abs(q[1, :2, 0] - bias).max() > 1e-3
    np.testing.assert_array_equal(hT[3], h0[3])
    assert np.abs(hT[:3] - h0[:3]).max() > 1e-3


def test_double_q_argmax_ties_go_to_the_lowest_index():
    x = torch.tensor([[1.0, 3.0, 3.0, -999999.0], [-999999.0, -999999.0, -999999.0, -999999.0], [2.0, 0.0, 2.0, 5.0]])
    assert qo.first_argmax(x).tolist() == [1, 0, 3]


def test_count_ties_counts_available_maxima_of_the_next_step_on_masked_in_rows():
    q = np.zeros((1, 3, 2, 4))
    avail = np.ones((1, 3, 2, 4))
    q[0, 1, 0] = [5, 5, 1, 0]                          # step 0, agent 0: tie
    q[0, 1, 1] = [5, 5, 9, 0]
    avail[0, 1, 1, 2] = 0                              # agent 1: the 9 is unavailable, so 5 and 5 tie
    q[0, 2, 0] = [1, 7, 7, 7]
    avail[0, 2, 0, 1:3] = 0                            # step 1, agent 0: one 7 left available, no tie
    q[0, 2, 1] = [2, 2, 0, 0]                          # step 1, agent 1: tie, but the row is masked out below
    assert qo.count_ties(q, avail, np.array([[1.0, 1.0]])) == 3
    assert qo.count_ties(q, avail, np.array([[1.0, 0.0]])) == 2
    avail[0, 1] = 0                                    # all unavailable (padding): nothing to break
    assert qo.count_ties(q, avail, np.array([[1.0, 0.0]])) == 0


def test_loss_gradient_matches_finite_differences():
    rng = np.random.default_rng(2)
    B, L, n, A, obs_dim, sd, H, E, he = 2, 4, 2, 3, 5, 6, 4, 3, 5
    w = _weights(rng, obs_dim, H, A, n, E, he, sd)
    wt = _weights(rng, obs_dim, H, A, n, E, he, sd)
    batch = qo.synth_batch(3, B, L, n, A, obs_dim, sd, max_ep_t=4)
    for double_q in (True, False):
        with orc.precision("f64"):
            wv = {k: qo._t(v).requires_grad_(True) for k, v in w.items()}
            wtv = {k: qo._t(v) for k, v in wt.items()}
            loss = qo.td_loss(wv, wtv, batch, 0.99, double_q)
            grads = torch.autograd.grad(loss, list(wv.values()), allow_unused=True)
            for (name, p), g in zip(wv.items(), grads):
                idx = tuple(rng.integers(0, s) for s in p.shape)
                eps = 1e-6
                with torch.no_grad():
                    base = p[idx].item()
                    p[idx] = base + eps
                    lp = float(qo.td_loss(wv, wtv, batch, 0.99, double_q))
                    p[idx] = base - eps
                    lm = float(qo.td_loss(wv, wtv, batch, 0.99, double_q))
                    p[idx] = base
                fd = (lp - lm) / (2 * eps)
                an = 0.0 if g is None else float(g[idx])
                assert abs(fd - an) <= 1e-6 * max(1.0, abs(fd)), (name, double_q, fd, an)


def test_synth_batch_mask_follows_the_reference_rule():
    b = qo.synth_batch(4, 4, 6, 2, 5, 3, 4, max_ep_t=5)
    filled = np.abs(b["obs"]).sum(axis=(2, 3)) > 0            # [B, L+1]: the steps an episode filled (obs are nonzero)
    want = filled[:, :-1].astype(np.float32)
    want[:, 1:] = want[:, 1:] * (1 - b["terminated"][:, :-1])
    assert b["terminated"].sum() > 0 and filled.sum() < filled.size
    np.testing.assert_array_equal(b["mask"], want)
