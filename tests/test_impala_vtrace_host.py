"""The float64 V-trace of the oracle, the yardstick of tests/test_gpu_impala_vtrace.py, on the CPU: under precision("f64")
vtrace_from_logits is the naive Espeholt et al. recursion in float64, and the autograd gradients of impala_loss are the
closed forms vtrace_kernel implements; the default precision still returns float32."""
import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc


def _naive_vtrace(bp, tp, act, disc, rew, val, boot):
    """v_s = V_s + delta_s + gamma_s c_s (v_{s+1} - V_{s+1}) (Espeholt et al. 2018, eq. 1), rho and c clipped at 1,
    one step at a time in float64"""
    lsm = lambda x: x - np.log(np.exp(x - x.max(-1, keepdims=True)).sum(-1, keepdims=True)) - x.max(-1, keepdims=True)  # noqa: E731
    pick = lambda x: np.take_along_axis(lsm(x.astype(np.float64)), act[..., None].astype(np.int64), -1)[..., 0]  # noqa: E731
    c = np.minimum(1.0, np.exp(pick(tp) - pick(bp)))
    T = val.shape[0]
    vs = np.zeros((T + 1,) + val.shape[1:])
    vs[T] = boot
    nv = np.concatenate([val[1:], boot[None]], 0)
    for t in range(T - 1, -1, -1):
        vs[t] = val[t] + c[t] * (rew[t] + disc[t] * nv[t] - val[t]) + disc[t] * c[t] * (vs[t + 1] - nv[t])
    return vs[:T], c * (rew + disc * vs[1:] - val)


def _inputs(T, B, A, seed, gamma):
    rng = np.random.default_rng(seed)
    tp = rng.standard_normal((T, B, A))
    bp = tp + 0.5 * rng.standard_normal((T, B, A))
    act = rng.integers(0, A, (T, B))
    disc = (rng.random((T, B)) > 0.1) * gamma
    return bp, tp, act, disc, rng.standard_normal((T, B)), rng.standard_normal((T, B)), rng.standard_normal(B)


@pytest.mark.parametrize("T,B,A,gamma", [(1, 1, 4, 0.99), (9, 3, 4, 0.99), (33, 5, 1, 0.99), (100, 2, 18, 1.0), (40, 4, 6, 0.0)])
def test_float64_vtrace_is_the_naive_recursion(T, B, A, gamma):
    args = _inputs(T, B, A, T * 100 + A, gamma)
    with orc.precision("f64"):
        vs, pg = orc.vtrace_from_logits(*args)
    assert vs.dtype == np.float64 and pg.dtype == np.float64
    vs_ref, pg_ref = _naive_vtrace(*args)
    np.testing.assert_allclose(vs, vs_ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(pg, pg_ref, rtol=1e-12, atol=1e-12)
    # fp32 inputs are widened, not computed in fp32: the same float64 result from the fp32-rounded values
    a32 = [x.astype(np.float32) if x.dtype == np.float64 else x for x in args]
    with orc.precision("f64"):
        vs32in, _ = orc.vtrace_from_logits(*a32)
    np.testing.assert_allclose(vs32in, _naive_vtrace(*[x.astype(np.float64) for x in a32])[0], rtol=1e-12, atol=1e-12)
    # the default precision is the reference's own fp32
    v, p = orc.vtrace_from_logits(*a32)
    assert v.dtype == np.float32 and p.dtype == np.float32


@pytest.mark.parametrize("k,S,A", [(1, 2, 4), (3, 17, 1), (2, 40, 6)])
def test_float64_impala_loss_gradients_are_the_kernel_closed_forms(k, S, A):
    """dL/dlogit_i = pg (p_i - [i = a]) + 0.01 p_i (log p_i + H), dL/dV_t = 0.5 (V_t - vs_t) on the kept rows, zero on
    row S - 1 of each trajectory (vs and pg are stop-gradient, so finite differences cannot check this)"""
    rng = np.random.default_rng(k * 10 + S)
    N, T = k * S, S - 1
    tp = rng.standard_normal((N, A)) * 2
    bp = (tp + 0.5 * rng.standard_normal((N, A))).astype(np.float32)
    base = rng.standard_normal(N)
    act = rng.integers(0, A, N).astype(np.int32)
    done = rng.random(N) < 0.1
    rew = (rng.standard_normal(N) * 2).astype(np.float32)
    gamma = float(np.float32(0.99))
    with orc.precision("f64"):
        tpt = torch.from_numpy(tp).requires_grad_(True)
        bt = torch.from_numpy(base).requires_grad_(True)
        loss = orc.impala_loss(tpt, bt, bp, act, done, rew, S, gamma=gamma)
        assert loss.dtype == torch.float64
        loss.backward()
        sb = lambda x: orc.split_batches(x, S, True)  # noqa: E731
        vs, pg = orc.vtrace_from_logits(sb(bp), sb(tp), sb(act), sb((~done) * gamma), sb(np.clip(rew, -1, 1)), sb(base),
                                        orc.split_batches(base, S)[-1])
    assert vs.dtype == np.float64 and pg.dtype == np.float64
    # time-major [T, k] -> env-major rows [k, S) with row S - 1 zero
    rows = lambda x: np.concatenate([np.asarray(x).T, np.zeros((k, 1))], 1).reshape(N)  # noqa: E731
    vs_r, pg_r = rows(vs), rows(pg)
    lsm = tp - tp.max(-1, keepdims=True)
    lsm = lsm - np.log(np.exp(lsm).sum(-1, keepdims=True))
    p = np.exp(lsm)
    H = -(p * lsm).sum(-1, keepdims=True)
    want_dl = pg_r[:, None] * (p - np.eye(A)[act]) + 0.01 * p * (lsm + H)
    want_db = 0.5 * (base - vs_r)
    last = np.arange(N) % S == S - 1
    want_dl[last] = 0.0
    want_db[last] = 0.0
    np.testing.assert_allclose(tpt.grad.numpy(), want_dl, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(bt.grad.numpy(), want_db, rtol=1e-12, atol=1e-12)
    assert not tpt.grad.numpy()[last].any() and not bt.grad.numpy()[last].any()
