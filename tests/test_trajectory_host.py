"""CPU tier: the trajectory yardsticks of tests/test_gpu_trajectory.py.

- orc.gae_f32 (GAE's backward loop in float32, vectorised over rows) equals a per-step float32 loop bit for bit, and
  orc.gae (float64) still equals the reference's own output in tests/golden/gae.npz;
- sign_clip_f32 is np.sign: +-1, +0 for both zeros, NaN kept; a NaN reward turns its own and every earlier advantage
  NaN in both restatements, across terminal steps;
- orc.nstep_returns equals a per-step loop bit for bit in float64 and float32, and gives the hand-worked windows of
  n >= T, a terminal last step, every step terminal and n = 1."""
import os

import numpy as np
import pytest

from oracle import xt_oracle as orc

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gae_loop_f32(value, reward, done, gamma, lam):
    """one trajectory, one step at a time, every operation rounded to float32"""
    f = np.float32
    T = len(reward)
    adv = np.zeros(T, f)
    nxt = f(0)
    for t in range(T - 1, -1, -1):
        disc = f(0) if done[t] else f(gamma)
        delta = f(f(f(reward[t]) + f(disc * f(value[t + 1]))) - f(value[t]))
        nxt = f(delta + f(f(disc * f(lam)) * nxt))
        adv[t] = nxt
    return adv


def _nstep_loop(reward, done, n, gamma, f):
    """one segment, one window at a time"""
    T = len(reward)
    ret = np.zeros(T, f); disc = np.zeros(T, f); last = np.zeros(T, np.int64); dn = np.zeros(T, bool)
    for t in range(T):
        acc, g, k, term = f(0), f(1), 0, False
        while k < n and t + k < T:
            acc = f(acc + f(g * f(reward[t + k])))
            g = f(g * f(gamma))
            k += 1
            if done[t + k - 1]:
                term = True
                break
        ret[t], disc[t], last[t], dn[t] = acc, (f(0) if term else g), t + k - 1, term
    return ret, disc, last, dn


def _rollout(rng, E, T, p_done):
    value = rng.standard_normal((E, T + 1)).astype(np.float32)
    reward = (2 * rng.standard_normal((E, T))).astype(np.float32)
    done = rng.random((E, T)) < p_done
    return value, reward, done


@pytest.mark.parametrize("E,T,gamma,lam,p_done", [(1, 1, 0.99, 0.95, 0.0), (3, 33, 0.99, 0.95, 0.1), (2, 64, 1.0, 1.0, 0.0),
                                                  (4, 17, 0.0, 0.95, 0.2), (2, 40, 0.99, 0.0, 0.1), (3, 9, 0.99, 0.95, 1.0)])
def test_gae_f32_equals_a_per_step_loop(E, T, gamma, lam, p_done):
    rng = np.random.default_rng(E * 100 + T)
    value, reward, done = _rollout(rng, E, T, p_done)
    adv, ov, tv = orc.gae_f32(value, reward, done, gamma, lam)
    assert adv.dtype == ov.dtype == tv.dtype == np.float32 and adv.shape == (E, T)
    for e in range(E):
        np.testing.assert_array_equal(adv[e], _gae_loop_f32(value[e], reward[e], done[e], gamma, lam))
    np.testing.assert_array_equal(ov, value[:, :T])
    np.testing.assert_array_equal(tv, adv + value[:, :T])
    # a [T + 1, 1] value column (the agent's layout) gives the same
    np.testing.assert_array_equal(orc.gae_f32(value[0][:, None], reward[0], done[0], gamma, lam)[0], adv[0])


def test_gae_against_the_reference_fixture():
    """orc.gae is the reference's float64 data_proc bit for bit; the float32 loop stays within fp32 rounding of it"""
    z = np.load(os.path.join(G, "gae.npz"))
    for c in range(6):
        value, reward, done = z["c%d_value" % c], z["c%d_reward" % c], z["c%d_done" % c]
        adv, ov, tv = orc.gae(value, reward, done)
        assert adv.dtype == np.float64
        np.testing.assert_array_equal(adv, z["c%d_adv" % c])
        np.testing.assert_array_equal(tv, z["c%d_target_value" % c])
        a32 = orc.gae_f32(value, reward, done)[0]
        scale = max(1.0, float(np.abs(z["c%d_adv" % c]).max()))
        assert np.abs(a32 - z["c%d_adv" % c][:, 0]).max() <= 1e-5 * scale, c


def test_sign_clip_is_np_sign():
    r = np.array([2.5, -0.25, 0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1.0, -1.0], np.float32)
    got, want = orc.sign_clip_f32(r), np.sign(r)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, want)                       # NaN where np.sign has NaN
    np.testing.assert_array_equal(np.signbit(got), np.signbit(want))
    assert not np.signbit(got[3]) and not np.signbit(np.sign(np.float32(-0.0)))   # -0 clips to +0


def test_sign_clipped_gae_and_nan_propagation():
    """gae_f32(sign_clip) is gae_f32 of np.sign(reward); a NaN reward makes its own step and every earlier step of the
    trajectory NaN, terminal steps in between or not, in float32 and in float64 alike"""
    rng = np.random.default_rng(7)
    E, T = 3, 40
    value, reward, done = _rollout(rng, E, T, 0.15)
    reward[:, ::5] = 0.0
    reward[:, 1::5] = -0.0
    reward[0, 30] = np.nan                    # a NaN with terminal steps before it
    done[0, 10] = done[0, 20] = True
    reward[2, 0] = np.nan                     # a NaN on the first step only
    a_clip = orc.gae_f32(value, reward, done, sign_clip=True)
    a_sign = orc.gae_f32(value, np.sign(reward), done)
    for x, y in zip(a_clip, a_sign):
        np.testing.assert_array_equal(x, y)
    want = np.zeros((E, T), bool)
    want[0, :31] = True
    want[2, 0] = True
    np.testing.assert_array_equal(np.isnan(a_clip[0]), want)
    np.testing.assert_array_equal(np.isnan(a_clip[2]), want)
    with np.errstate(invalid="ignore"):
        for e in range(E):
            a64, _, t64 = orc.gae(value[e][:, None], np.sign(reward[e]).astype(np.float64), done[e])
            np.testing.assert_array_equal(np.isnan(a64[:, 0]), want[e])
            np.testing.assert_array_equal(np.isnan(t64[:, 0]), want[e])


@pytest.mark.parametrize("E,T,n,gamma,p_done", [(1, 1, 1, 0.99, 0.0), (5, 33, 3, 0.99, 0.1), (2, 10, 12, 1.0, 0.0),
                                                (3, 20, 19, 0.0, 0.2), (4, 16, 5, 0.99, 1.0), (2, 50, 50, 0.99, 0.05)])
def test_nstep_returns_equal_a_per_step_loop(E, T, n, gamma, p_done):
    rng = np.random.default_rng(E * 1000 + T * 10 + n)
    reward = (2 * rng.standard_normal((E, T))).astype(np.float32)
    done = rng.random((E, T)) < p_done
    done[0, T - 1] = True
    for f in (np.float64, np.float32):
        ret, disc, last, dn = orc.nstep_returns(reward, done, n, gamma, dtype=f)
        assert ret.dtype == disc.dtype == f and ret.shape == disc.shape == last.shape == dn.shape == (E, T)
        for e in range(E):
            r_ret, r_disc, r_last, r_dn = _nstep_loop(reward[e], done[e], n, gamma, f)
            np.testing.assert_array_equal(ret[e], r_ret)
            np.testing.assert_array_equal(disc[e], r_disc)
            np.testing.assert_array_equal(last[e], r_last + e * T)    # flat row indices across segments
            np.testing.assert_array_equal(dn[e], r_dn)


NSTEP_HAND = [
    # name, reward, done, n, gamma: ret, disc, last, done_n
    ("n_ge_T", [1, 2, 3], [0, 0, 0], 5, 0.5, [2.75, 3.5, 3.0], [0.125, 0.25, 0.5], [2, 2, 2], [0, 0, 0]),
    ("done_last", [1, 2, 3], [0, 0, 1], 2, 0.5, [2.0, 3.5, 3.0], [0.25, 0.0, 0.0], [1, 2, 2], [0, 1, 1]),
    ("all_done", [1, 2, 3], [1, 1, 1], 3, 0.5, [1.0, 2.0, 3.0], [0.0, 0.0, 0.0], [0, 1, 2], [1, 1, 1]),
    ("n1", [1, 2, 3], [0, 1, 0], 1, 0.5, [1.0, 2.0, 3.0], [0.5, 0.0, 0.5], [0, 1, 2], [0, 1, 0]),
    ("n_eq_T_done_mid", [1, 2, 3, 4], [0, 1, 0, 0], 4, 0.5, [2.0, 2.0, 5.0, 4.0], [0.0, 0.0, 0.25, 0.5], [1, 1, 3, 3], [1, 1, 0, 0]),
]


@pytest.mark.parametrize("case", NSTEP_HAND, ids=[c[0] for c in NSTEP_HAND])
def test_nstep_returns_hand_worked(case):
    _, reward, done, n, gamma, ret, disc, last, dn = case
    got = orc.nstep_returns(np.array(reward, np.float32), np.array(done, bool), n, gamma)
    np.testing.assert_array_equal(got[0], ret)
    np.testing.assert_array_equal(got[1], disc)
    np.testing.assert_array_equal(got[2], last)
    np.testing.assert_array_equal(got[3], np.array(dn, bool))


def test_nstep_returns_last_is_flat_across_segments():
    """two segments of two steps, windows of three: each window stops at its own segment's end"""
    ret, disc, last, dn = orc.nstep_returns(np.ones((2, 2), np.float32), np.zeros((2, 2), bool), 3, 0.5)
    np.testing.assert_array_equal(last, [[1, 1], [3, 3]])
    np.testing.assert_array_equal(ret, [[1.5, 1.0], [1.5, 1.0]])
    np.testing.assert_array_equal(disc, [[0.25, 0.5], [0.25, 0.5]])
    assert not dn.any()
