"""The trajectory kernels that build the learners' targets, against float64:

a. gae_kernel through xtb_gae: adv and target_v against the oracle's float64 GAE at the trajectory lengths where the
   warp's lane chunks change (chunk = (T + 31) / 32 steps per lane), env counts that fill the last 128-thread block with
   one to four warps, (gamma, lam) with and without decay, no / every / random terminal steps and terminal steps on both
   edges of every lane's chunk (where the chunk's composed map is x -> 0 x + b), sign-clipped rewards, and values of
   1e4 next to small rewards; old_v bit for bit.  Its contract: every output written, an empty rollout a no-op, a
   negative size or a null pointer refused without a launch.  A NaN reward under sign_clip turns the advantages NaN
   exactly where the reference's GAE on np.sign(reward) has them;
b. nstep_kernel through xtb_nstep_returns: ret and disc against float64, last and done_n exactly, over several blocks
   with segment boundaries inside a block and windows shorter than, equal to and longer than the segment;
c. argmax_kernel through xtb_argmax: exactly np.argmax, ties, rows of -inf and NaN included;
d. the learner-side data paths: PPO's device GAE over raw trajectories of equal and unequal lengths, mixed with
   precomputed ones, sign-clipped, and across a growth of its raw stores; DQN's n-step transitions in its replay ring,
   across a wrap of the ring and a segment shorter than n.

fp32 results are held to K times the distance of a plain float32 restatement (orc.gae_f32, orc.nstep_returns in
float32) from float64, plus a floor of a few fp32 ulps.  Every observed error is recorded through
tests/parity_record.py."""
import collections

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from parity_record import record
from test_gpu_kernels import _keepalive, dev, rel_err, xb  # noqa: F401

pytestmark = pytest.mark.gpu

XTB_ERR_ARG = -1
K = 4
# about four fp32 ulps (relative to the largest reference magnitude) on top of K x the fp32 restatement's distance from
# float64 (observed on an NVIDIA H100 80GB HBM3 at 700 W: at most 23 % of the bound, on PPO's target_v of four raw
# 50-step trajectories; the kernels alone at most 21 %, GAE at T = 4096 with gamma = lam = 1, where the device is 7.7e-7
# from float64 and the fp32 restatement 7.9e-7; the device error at most 1.3 x the restatement's on the kernels)
FLOOR = 5e-7


def _f32(x):
    """the value a C float argument carries"""
    return float(np.float32(x))


def _within(name, errs):
    """errs: {output: (device error, fp32 restatement error)}; records them and returns the outputs over the bound"""
    record(name, {k: ["%.2e" % a, "%.2e" % b, "%.1f%%" % (100 * a / (K * b + FLOOR))] for k, (a, b) in errs.items()})
    return {k: e for k, e in errs.items() if not e[0] <= K * e[1] + FLOOR}


@pytest.fixture(autouse=True)
def _restore_module_config():
    """import_config writes the algorithm and model configs into their modules' globals: restore them"""
    from xingtian_b200.algorithm import dqn as alg_dqn, ppo as alg_ppo
    from xingtian_b200.model import dqn as model_dqn, ppo as model_ppo
    mods = (alg_dqn, alg_ppo, model_dqn, model_ppo)
    saved = [{k: v for k, v in vars(m).items() if k.isupper()} for m in mods]
    yield
    for m, s in zip(mods, saved):
        for k in [k for k in vars(m) if k.isupper() and k not in s]:
            delattr(m, k)
        for k, v in s.items():
            setattr(m, k, v)


def _launches(xb):
    torch.cuda.synchronize()
    return xb["lib"].xtb_launch_count()


# ---- a. xtb_gae -----------------------------------------------------------------------------------------------------
class GCase(collections.namedtuple("GCase", "E T gamma lam dones clip big")):
    """E envs of T steps; dones: "none", "all", "random" (~5 %) or "edges" (the first and the last step of every lane's
    chunk); clip: sign_clip; big: |V| ~ 1e4 with rewards ~ 1e-2"""

    @property
    def id(self):
        return "E%d-T%d-g%g-l%g-%s%s%s" % (self.E, self.T, self.gamma, self.lam, self.dones, "-clip" if self.clip else "",
                                           "-big" if self.big else "")


GAE = [
    # T = 1 and 2: one and two lanes busy; T = 31 / 32: one step per lane, 31 or 32 lanes; T = 33: 17 lanes of two steps
    GCase(1, 1, 0.99, 0.95, "none", 0, False), GCase(3, 2, 0.99, 0.95, "all", 1, False),
    GCase(4, 31, 0.99, 0.95, "random", 0, False), GCase(5, 32, 0.99, 0.95, "edges", 1, False),
    GCase(1, 33, 1.0, 1.0, "none", 0, False), GCase(4, 33, 0.0, 0.95, "all", 0, False),
    # T = 63 / 64 / 65: chunks of 2, 2 and 3 steps; the last busy lane's chunk partly filled at 63 and 65
    GCase(3, 63, 0.0, 0.95, "random", 1, False), GCase(4, 64, 0.99, 0.0, "random", 0, False),
    GCase(5, 65, 0.99, 0.95, "edges", 0, False), GCase(512, 65, 1.0, 1.0, "random", 0, False),
    # the C5 shape, 512 x 128, with and without sign_clip; T = 129: chunks of 5, the 26th lane with four steps
    GCase(512, 128, 0.99, 0.95, "random", 1, False), GCase(512, 128, 0.99, 0.95, "random", 0, True),
    GCase(4, 128, 1.0, 1.0, "edges", 1, False), GCase(3, 129, 1.0, 1.0, "random", 0, False),
    GCase(5, 129, 0.99, 0.0, "none", 1, False),
    # long trajectories: chunks of 32 and 128 steps; (1, 1) without terminal steps sums over the whole trajectory
    GCase(1, 1000, 0.99, 0.95, "random", 0, True), GCase(5, 1000, 1.0, 1.0, "none", 0, False),
    GCase(3, 1000, 0.99, 0.95, "all", 1, False), GCase(3, 4096, 1.0, 1.0, "none", 0, False),
    GCase(1, 4096, 0.99, 0.95, "edges", 1, False), GCase(5, 4096, 0.99, 0.95, "random", 0, True),
]


def _gae_data(c):
    rng = np.random.default_rng(c.E * 100003 + c.T * 11 + int(c.gamma * 100) + int(c.lam * 10) + c.clip)
    E, T = c.E, c.T
    value = ((1e4 if c.big else 1.0) * rng.standard_normal((E, T + 1))).astype(np.float32)
    reward = ((1e-2 if c.big else 2.0) * rng.standard_normal((E, T))).astype(np.float32)
    if c.clip:
        reward[:, 0::7], reward[:, 3::7], reward[:, 5::7], reward[:, 6::7] = 0.0, -0.0, 1.0, -1.0
    done = np.zeros((E, T), bool)
    if c.dones == "all":
        done[:] = True
    elif c.dones == "random":
        done = rng.random((E, T)) < 0.05
    elif c.dones == "edges":
        chunk = (T + 31) // 32
        done[:, 0::chunk] = True
        done[:, chunk - 1::chunk] = True
        done[:, T - 1] = True
    return value, reward, done


def _assert_gae_regimes(c, value, reward, done):
    """each regime the case is named for occurs in its data"""
    if c.dones == "none":
        assert not done.any()
    elif c.dones == "all":
        assert done.all()
    elif c.dones == "random":
        assert done.any() and not done.all()
    else:
        chunk = (c.T + 31) // 32
        for t0 in range(0, c.T, chunk):
            assert done[:, t0].all() and done[:, min(c.T, t0 + chunk) - 1].all()
    if c.clip and c.T >= 7:
        r = reward
        assert (np.abs(r) > 1).any() and (r == 1).any() and (r == -1).any()
        assert ((r == 0) & ~np.signbit(r)).any() and ((r == 0) & np.signbit(r)).any()
    if c.big:
        assert np.abs(value).max() > 1e4 and np.abs(reward).max() < 0.1


def _gae_f64(value, reward, done, gamma, lam, clip):
    """the reference's float64 GAE per env on the rewards the kernel reads (np.sign of them under sign_clip)"""
    r = np.sign(reward) if clip else reward
    out = [orc.gae(value[e][:, None], r[e].astype(np.float64), done[e], _f32(gamma), _f32(lam)) for e in range(len(value))]
    return np.stack([a[:, 0] for a, _, _ in out]), np.stack([tv[:, 0] for _, _, tv in out])


def _gae_bufs(E, T, fill=float("nan")):
    return [torch.full((max(E, 1), max(T, 1)), fill, device="cuda") for _ in range(3)]


def _run_gae(xb, value, reward, done, gamma, lam, clip):
    """xtb_gae into NaN-prefilled outputs: (adv, old_v, target_v) on the host"""
    from xingtian_b200.engine import _ptr, stream_ptr
    E, T = reward.shape
    adv, ov, tv = _gae_bufs(E, T)
    xb["capi"].check(xb["lib"].xtb_gae(_ptr(dev(value)), _ptr(dev(reward)), _ptr(dev(done.view(np.uint8))), E, T, gamma, lam,
                                      int(clip), _ptr(adv), _ptr(ov), _ptr(tv), stream_ptr()))
    torch.cuda.synchronize()
    return adv.cpu().numpy(), ov.cpu().numpy(), tv.cpu().numpy()


@pytest.mark.parametrize("c", GAE, ids=[c.id for c in GAE])
def test_gae_against_float64(xb, c):
    """adv and target_v within K x the fp32 restatement's error + FLOOR of float64; old_v = value[:, :T] bit for bit;
    every output written"""
    value, reward, done = _gae_data(c)
    _assert_gae_regimes(c, value, reward, done)
    a64, t64 = _gae_f64(value, reward, done, c.gamma, c.lam, c.clip)
    a32, _, t32 = orc.gae_f32(value, reward, done, c.gamma, c.lam, sign_clip=c.clip)
    adv, ov, tv = _run_gae(xb, value, reward, done, c.gamma, c.lam, c.clip)
    for name, x in (("adv", adv), ("old_v", ov), ("target_v", tv)):
        assert not np.isnan(x).any(), name
    bad = _within("gae_vs_f64/%s" % c.id, {"adv": (rel_err(adv, a64), rel_err(a32, a64)),
                                           "target_v": (rel_err(tv, t64), rel_err(t32, t64))})
    assert not bad, bad
    np.testing.assert_array_equal(ov, value[:, :c.T])


def test_gae_sign_clip_keeps_nan(xb):
    """Under sign_clip a NaN reward is np.sign's NaN: adv and target_v are NaN at exactly the steps where the reference's
    float64 GAE on np.sign(reward) has NaN (the step and every earlier step of its trajectory, terminal steps in between
    or not), the rest within the bound.  Without sign_clip the same."""
    E, T = 4, 65                                      # chunks of 3 steps over 22 lanes
    rng = np.random.default_rng(11)
    value = rng.standard_normal((E, T + 1)).astype(np.float32)
    reward = (2 * rng.standard_normal((E, T))).astype(np.float32)
    reward[:, ::4] = 0.0
    done = rng.random((E, T)) < 0.1
    reward[0, 40] = np.nan                            # inside lane 13's chunk, terminal steps before it
    done[0, 39] = done[0, 12] = True
    reward[1, T - 1] = np.nan                         # the last step: the whole trajectory
    reward[2, 0] = np.nan                             # the first step only
    want = np.zeros((E, T), bool)
    want[0, :41] = want[1, :] = want[2, 0] = True
    for clip in (1, 0):
        with np.errstate(invalid="ignore"):
            a64, t64 = _gae_f64(value, reward, done, 0.99, 0.95, clip)
            a32, _, t32 = orc.gae_f32(value, reward, done, 0.99, 0.95, sign_clip=bool(clip))
        np.testing.assert_array_equal(np.isnan(a64), want)
        adv, ov, tv = _run_gae(xb, value, reward, done, 0.99, 0.95, clip)
        np.testing.assert_array_equal(np.isnan(adv), want, err_msg="adv, sign_clip=%d" % clip)
        np.testing.assert_array_equal(np.isnan(tv), want, err_msg="target_v, sign_clip=%d" % clip)
        np.testing.assert_array_equal(ov, value[:, :T])
        ok = ~want
        bad = _within("gae_vs_f64/nan-clip%d" % clip, {"adv": (rel_err(adv[ok], a64[ok]), rel_err(a32[ok], a64[ok])),
                                                       "target_v": (rel_err(tv[ok], t64[ok]), rel_err(t32[ok], t64[ok]))})
        assert not bad, bad


def test_gae_contract(xb):
    """an empty rollout (E = 0 or T = 0) is a no-op; a negative size and each null pointer are refused with a message and
    without a launch; the outputs are untouched by all of them"""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = xb["lib"]
    E, T = 3, 5
    ins = [dev(np.zeros((E, T + 1), np.float32)), dev(np.ones((E, T), np.float32)), dev(np.zeros((E, T), np.uint8))]
    outs = _gae_bufs(E, T, fill=7.0)

    def call(e, t, null=()):
        p = [None if i in null else _ptr(x) for i, x in enumerate(ins + outs)]
        return lib.xtb_gae(*p[:3], e, t, 0.99, 0.95, 0, *p[3:], stream_ptr())

    before = _launches(xb)
    for e, t in ((0, 0), (0, T), (E, 0)):
        assert call(e, t) == 0, (e, t)
    for e, t in ((-1, 0), (0, -1), (-1, T), (E, -1), (-5, -5)):
        assert call(e, t) == XTB_ERR_ARG, (e, t)
        assert b"xtb_gae: negative size" in lib.xtb_last_error(), (e, t)
    for i in range(6):
        assert call(E, T, null=(i,)) == XTB_ERR_ARG, i
        assert b"xtb_gae: null pointer" in lib.xtb_last_error(), i
    assert _launches(xb) == before
    for o in outs:
        assert (o.cpu().numpy() == 7.0).all()
    assert call(E, T) == 0
    assert _launches(xb) == before + 1


# ---- b. xtb_nstep_returns -------------------------------------------------------------------------------------------
class NCase(collections.namedtuple("NCase", "E T n gamma dones")):
    """E segments of T steps, windows of n; dones: "none", "all", "random" (~10 %) or "last" (each segment's last step)"""

    @property
    def id(self):
        return "E%d-T%d-n%d-g%g-%s" % (self.E, self.T, self.n, self.gamma, self.dones)


NSTEP = [
    # the shapes of the earlier test, (E, T, n) = (1, 64, 3), (5, 33, 1), (3, 40, 5)
    NCase(1, 64, 3, 0.99, "random"), NCase(5, 33, 1, 0.99, "random"), NCase(3, 40, 5, 0.99, "all"),
    # E = 5, T = 33: 165 rows over two blocks, segment boundaries inside both; n = T - 1, T, T + 7
    NCase(5, 33, 3, 1.0, "last"), NCase(5, 33, 5, 0.0, "none"), NCase(5, 33, 32, 0.99, "none"),
    NCase(5, 33, 33, 1.0, "random"), NCase(5, 33, 40, 0.99, "last"),
    # one step; one window longer than its segment
    NCase(1, 1, 1, 0.99, "none"), NCase(1, 1, 8, 0.99, "last"),
    # 903 rows (8 blocks); 1200 rows with n = T - 1; 1300 rows with n = T + 7; 5000 rows of five-step segments
    NCase(7, 129, 5, 1.0, "random"), NCase(4, 300, 299, 0.99, "random"), NCase(13, 100, 107, 1.0, "last"),
    NCase(1000, 5, 3, 0.99, "random"), NCase(9, 128, 128, 0.99, "none"), NCase(2, 2, 1, 0.0, "all"),
]


def _nstep_data(c):
    rng = np.random.default_rng(c.E * 1009 + c.T * 13 + c.n)
    reward = (2 * rng.standard_normal((c.E, c.T))).astype(np.float32)
    done = np.zeros((c.E, c.T), bool)
    if c.dones == "all":
        done[:] = True
    elif c.dones == "random":
        done = rng.random((c.E, c.T)) < 0.1
    elif c.dones == "last":
        done[:, -1] = True
    return reward, done


def _assert_nstep_regimes(c, done):
    if c.dones == "none":
        assert not done.any()
    elif c.dones == "all":
        assert done.all()
    elif c.dones == "random":
        assert done.any() and not done.all()
    else:
        assert done[:, -1].all() and not done[:, :-1].any()
    if c.E * c.T > 128:
        assert c.E > 1                         # several segments over several blocks


def _run_nstep(xb, reward, done, n, gamma):
    from xingtian_b200.engine import _ptr, stream_ptr
    E, T = reward.shape
    ret = torch.full((E, T), float("nan"), device="cuda"); disc = torch.full((E, T), float("nan"), device="cuda")
    last = torch.full((E, T), -1, dtype=torch.int32, device="cuda"); dn = torch.full((E, T), 7, dtype=torch.uint8, device="cuda")
    xb["capi"].check(xb["lib"].xtb_nstep_returns(_ptr(dev(reward)), _ptr(dev(done.view(np.uint8))), E, T, n, gamma, _ptr(ret),
                                                _ptr(disc), _ptr(last), _ptr(dn), stream_ptr()))
    torch.cuda.synchronize()
    return ret.cpu().numpy(), disc.cpu().numpy(), last.cpu().numpy(), dn.cpu().numpy()


@pytest.mark.parametrize("c", NSTEP, ids=[c.id for c in NSTEP])
def test_nstep_against_float64(xb, c):
    """ret and disc within K x the fp32 restatement's error + FLOOR of float64; last (flat rows) and done_n exactly"""
    reward, done = _nstep_data(c)
    _assert_nstep_regimes(c, done)
    r64, d64, l64, n64 = orc.nstep_returns(reward, done, c.n, _f32(c.gamma))
    r32, d32, _, _ = orc.nstep_returns(reward, done, c.n, _f32(c.gamma), dtype=np.float32)
    ret, disc, last, dn = _run_nstep(xb, reward, done, c.n, c.gamma)
    assert not np.isnan(ret).any() and not np.isnan(disc).any()
    bad = _within("nstep_vs_f64/%s" % c.id, {"ret": (rel_err(ret, r64), rel_err(r32, r64)),
                                             "disc": (rel_err(disc, d64), rel_err(d32, d64))})
    assert not bad, bad
    np.testing.assert_array_equal(last, l64)
    np.testing.assert_array_equal(dn, n64.astype(np.uint8))


def test_nstep_contract(xb):
    """a size below 1 or a null pointer is refused with a message and without a launch"""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = xb["lib"]
    E, T = 2, 4
    bufs = [dev(np.zeros((E, T), np.float32)), dev(np.zeros((E, T), np.uint8)), dev(np.zeros((E, T), np.float32)),
            dev(np.zeros((E, T), np.float32)), dev(np.zeros((E, T), np.int32)), dev(np.zeros((E, T), np.uint8))]

    def call(e=E, t=T, n=3, null=()):
        p = [None if i in null else _ptr(x) for i, x in enumerate(bufs)]
        return lib.xtb_nstep_returns(p[0], p[1], e, t, n, 0.99, *p[2:], stream_ptr())

    before = _launches(xb)
    for kw in (dict(e=0), dict(t=0), dict(n=0), dict(e=-1), dict(t=-1), dict(n=-1)):
        assert call(**kw) == XTB_ERR_ARG, kw
        assert b"xtb_nstep_returns: bad sizes" in lib.xtb_last_error(), kw
    for i in range(6):
        assert call(null=(i,)) == XTB_ERR_ARG, i
        assert b"xtb_nstep_returns: null pointer" in lib.xtb_last_error(), i
    assert _launches(xb) == before
    assert call() == 0 and _launches(xb) == before + 1


# ---- c. xtb_argmax --------------------------------------------------------------------------------------------------
ARGMAX = [(B, A) for B in (1, 127, 128, 129, 4096) for A in (1, 2, 18, 33)]
ROW_KINDS = ("plain", "tie", "all_neg_inf", "nan_first", "nan_later", "two_nans", "inf", "constant")


def _argmax_data(B, A):
    """row b is of kind ROW_KINDS[b % 8] (A = 1: plain, all -inf or NaN)"""
    rng = np.random.default_rng(B * 37 + A)
    q = rng.standard_normal((B, A)).astype(np.float32)
    for b in range(B):
        kind = ROW_KINDS[b % len(ROW_KINDS)]
        if kind == "all_neg_inf":
            q[b] = -np.inf
        elif kind == "nan_first":
            q[b, 0] = np.nan
        elif A < 2:
            continue
        elif kind == "tie":                       # two equal maxima: the first wins
            i, j = sorted(rng.choice(A, 2, replace=False))
            q[b, i] = q[b, j] = q[b].max() + 1.0
        elif kind == "nan_later":                 # the row's maximum at 0, a NaN after it
            q[b, 0] = q[b].max() + 1.0
            q[b, int(rng.integers(1, A))] = np.nan
        elif kind == "two_nans":
            i, j = sorted(rng.choice(np.arange(1, A), 2, replace=False)) if A > 2 else (1, 1)
            q[b, i] = np.nan
            q[b, j] = -np.nan
        elif kind == "inf":
            q[b, int(rng.integers(1, A))] = np.inf
            q[b, 0] = -np.inf
        elif kind == "constant":
            q[b] = 0.5
    return q


def _run_argmax(xb, q):
    from xingtian_b200.engine import _ptr, stream_ptr
    B, A = q.shape
    act = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    xb["capi"].check(xb["lib"].xtb_argmax(_ptr(dev(q)), B, A, _ptr(act), stream_ptr()))
    torch.cuda.synchronize()
    return act.cpu().numpy()


@pytest.mark.parametrize("B,A", ARGMAX, ids=["B%d-A%d" % s for s in ARGMAX])
def test_argmax_is_np_argmax(xb, B, A):
    """exactly np.argmax: the first maximum, the first NaN, 0 for a row of -inf"""
    q = _argmax_data(B, A)
    want = np.argmax(q, axis=1)
    if B >= 127 and A >= 2:
        kinds = np.arange(B) % len(ROW_KINDS)
        tie = kinds == ROW_KINDS.index("tie")
        assert ((q[tie] == q[tie].max(1, keepdims=True)).sum(1) == 2).all()
        nan_later = kinds == ROW_KINDS.index("nan_later")
        assert (want[nan_later] > 0).all() and np.isnan(q[nan_later]).any(1).all()
        if A > 2:
            assert (np.isnan(q).sum(1) == 2).any()
        assert np.isneginf(q).all(1).any() and np.isnan(q[:, 0]).any() and np.isposinf(q).any()
    np.testing.assert_array_equal(_run_argmax(xb, q), want)


def test_argmax_first_nan_wins(xb):
    """a NaN anywhere in the row is the row's argmax, as np.argmax picks it (the first NaN when there are several)"""
    q = np.array([[0.0, 1.0, np.nan, 3.0, 2.0],
                  [5.0, 1.0, 2.0, 3.0, np.nan],
                  [-np.inf, np.nan, np.inf, np.nan, 0.0],
                  [np.nan, 9.0, np.nan, 1.0, 2.0],
                  [1.0, 1.0, -np.nan, 1.0, 1.0],
                  [-np.inf, -np.inf, -np.inf, -np.inf, np.nan]], np.float32)
    want = np.argmax(q, axis=1)
    np.testing.assert_array_equal(want, [2, 4, 1, 0, 2, 4])
    np.testing.assert_array_equal(_run_argmax(xb, q), want)


def test_argmax_refuses_bad_arguments(xb):
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = xb["lib"]
    q, act = dev(np.zeros((4, 3), np.float32)), dev(np.zeros(4, np.int32))
    before = _launches(xb)
    for args in ((None, 4, 3, _ptr(act)), (_ptr(q), 4, 3, None), (_ptr(q), 0, 3, _ptr(act)), (_ptr(q), 4, 0, _ptr(act)),
                 (_ptr(q), -1, 3, _ptr(act))):
        assert lib.xtb_argmax(*args, stream_ptr()) == XTB_ERR_ARG
        assert b"xtb_argmax: bad argument" in lib.xtb_last_error()
    assert _launches(xb) == before


# ---- d. the learner-side data paths ---------------------------------------------------------------------------------
def _ppo_alg(sign_clip=False):
    import xingtian_b200 as xbp
    info = {"actor": {"model_name": "PpoMlp", "state_dim": [4], "action_dim": 2, "input_dtype": "float32",
                      "model_config": {"BATCH_SIZE": 64, "NUM_SGD_ITER": 1, "LR": 0.0003, "SUMMARY": False, "VF_SHARE_LAYERS": False,
                                       "activation": "tanh", "hidden_sizes": [32, 32], "action_type": "Categorical", "init_seed": 2}}}
    cfg = {"instance_num": 4, "agent_num": 1}
    if sign_clip:
        cfg["sign_clip_reward"] = True
    return xbp.alg_builder("PPO", info, cfg)


def _ppo_traj(rng, T, raw, clip=False):
    value = rng.standard_normal(T + 1).astype(np.float32)
    reward = (2 * rng.standard_normal(T)).astype(np.float32)
    if clip:
        reward[::5], reward[1::5], reward[2::5] = 0.0, -0.0, 1.0
    done = rng.random(T) < 0.08
    tr = dict(cur_state=rng.standard_normal((T, 4)).astype(np.float32), action=rng.integers(0, 2, T),
              logp=np.log(np.full((T, 1), 0.5, np.float32)), value=value, reward=reward, done=done, raw=raw)
    if not raw:   # the reference's message: advantages and targets from the explorer's float64 GAE
        adv, ov, tv = orc.gae(value[:, None], reward.astype(np.float64), done)
        tr.update(adv=adv, old_value=ov, target_value=tv)
    return tr


def _ppo_send(alg, trajs):
    for tr in trajs:
        keys = ("value", "reward", "done") if tr["raw"] else ("adv", "old_value", "target_value")
        alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp") + keys})


def _ppo_check(name, alg, trajs, clip=False):
    """the rollout's adv / old_v / target_v rows: raw trajectories against float64 GAE under the kernel bound, old_v bit for
    bit; precomputed ones exactly the float32 of what was sent"""
    ro = alg.actor.rollout
    n = sum(len(t["reward"]) for t in trajs)
    adv, ov, tv = (getattr(ro, k)[:n].cpu().numpy() for k in ("adv", "old_v", "target_v"))
    off, errs = 0, {}
    for i, tr in enumerate(trajs):
        T = len(tr["reward"])
        sl = slice(off, off + T)
        if tr["raw"]:
            a64, t64 = _gae_f64(tr["value"][None], tr["reward"][None], tr["done"][None], orc.GAMMA, orc.LAM, clip)
            a32, _, t32 = orc.gae_f32(tr["value"], tr["reward"], tr["done"], orc.GAMMA, orc.LAM, sign_clip=clip)
            errs["adv%d" % i] = (rel_err(adv[sl], a64[0]), rel_err(a32, a64[0]))
            errs["target_v%d" % i] = (rel_err(tv[sl], t64[0]), rel_err(t32, t64[0]))
            np.testing.assert_array_equal(ov[sl], tr["value"][:T])
        else:
            np.testing.assert_array_equal(adv[sl], tr["adv"][:, 0].astype(np.float32))
            np.testing.assert_array_equal(ov[sl], tr["old_value"][:, 0])
            np.testing.assert_array_equal(tv[sl], tr["target_value"][:, 0].astype(np.float32))
        off += T
    bad = _within("ppo_gae_vs_f64/%s" % name, errs)
    assert not bad, bad


PPO_LAYOUTS = {
    # name: [(T, raw)], the xtb_gae launches of the device GAE
    "equal_raw": ([(50, True)] * 4, 1),
    "unequal_raw": ([(1, True), (33, True), (200, True)], 3),
    "pre_then_raw": ([(20, False), (30, True), (30, True)], 1),
    "raw_then_pre": ([(30, True), (30, True), (20, False)], 1),
    "alternating": ([(17, True), (5, False), (17, True), (9, False), (17, True)], 3),
}


@pytest.mark.parametrize("layout", list(PPO_LAYOUTS))
def test_ppo_device_gae_layouts(xb, layout):
    """prepare_data + train() with raw trajectories (value[T+1], reward, done) among precomputed ones: one xtb_gae launch
    for equally long adjacent raw trajectories, one per trajectory otherwise, value offsets that skip the precomputed
    rows; the rollout's rows after the step are float64 GAE's"""
    shapes, launches = PPO_LAYOUTS[layout]
    rng = np.random.default_rng(len(layout) * 7 + len(shapes))
    trajs = [_ppo_traj(rng, T, raw) for T, raw in shapes]
    alg = _ppo_alg()
    _ppo_send(alg, trajs)
    before = _launches(xb)
    alg._device_gae()
    assert _launches(xb) - before == launches
    np.random.seed(0)
    assert np.isfinite(alg.train())
    _ppo_check(layout, alg, trajs)


def test_ppo_device_gae_sign_clip(xb):
    """sign_clip_reward: the device GAE of np.sign(reward), zeros of both signs included"""
    rng = np.random.default_rng(5)
    trajs = [_ppo_traj(rng, 64, True, clip=True) for _ in range(3)]
    assert any(((t["reward"] == 0) & np.signbit(t["reward"])).any() for t in trajs)
    alg = _ppo_alg(sign_clip=True)
    _ppo_send(alg, trajs)
    np.random.seed(0)
    assert np.isfinite(alg.train())
    _ppo_check("sign_clip", alg, trajs, clip=True)


def test_ppo_device_gae_across_store_growth(xb):
    """a second iteration with longer raw trajectories: the first reuses the raw stores of the first iteration, the later
    ones grow them (each growth keeps the rows already staged)"""
    rng = np.random.default_rng(9)
    alg = _ppo_alg()
    first = [_ppo_traj(rng, 40, True) for _ in range(2)]
    _ppo_send(alg, first)
    np.random.seed(0)
    alg.train()
    _ppo_check("grow/first", alg, first)
    cap = alg._raw_steps.capacity, alg._raw_values.capacity
    second = [_ppo_traj(rng, 60, True), _ppo_traj(rng, 60, False), _ppo_traj(rng, 60, True), _ppo_traj(rng, 70, True)]
    _ppo_send(alg, second[:1])
    assert (alg._raw_steps.capacity, alg._raw_values.capacity) == cap       # fits: reused
    _ppo_send(alg, second[1:])
    assert alg._raw_steps.capacity > cap[0] and alg._raw_values.capacity > cap[1]
    np.random.seed(0)
    alg.train()
    _ppo_check("grow/second", alg, second)


DQN_FEEDS = {
    # name: (N_STEP, GAMMA, BUFFER_SIZE, [(segment length, dones)])
    "n3_wrap": (3, 0.99, 100, [(50, "random"), (64, "random"), (2, "none"), (7, "last")]),
    "n5_wrap_short": (5, 1.0, 64, [(40, "last"), (90, "random"), (3, "none"), (4, "all")]),
}


@pytest.mark.parametrize("name", list(DQN_FEEDS))
def test_dqn_nstep_ring(xb, name):
    """prepare_data with N_STEP > 1 fills the replay ring with n-step transitions: reward and disc against float64 under
    the kernel bound, done and next_obs (the state after each window) exactly, across a wrap of the ring and with
    segments shorter than n"""
    import xingtian_b200 as xbp
    n, gamma, cap, segs = DQN_FEEDS[name]
    info = {"actor": {"model_name": "DqnMlp", "state_dim": [4], "action_dim": 2, "model_config": {"init_seed": 3}}}
    alg = xbp.alg_builder("DQN", info, {"instance_num": 1, "agent_num": 1, "BUFFER_SIZE": cap, "BATCH_SIZE": 8, "N_STEP": n,
                                         "GAMMA": gamma})
    assert alg.n_step == n
    rng = np.random.default_rng(n * 100 + cap)
    sent = []     # per transition, in the order sent: (obs, action, next_obs, seg, row)
    refs = []
    for si, (T, dones) in enumerate(segs):
        s = rng.standard_normal((T, 4)).astype(np.float32)
        s2 = rng.standard_normal((T, 4)).astype(np.float32)
        a = rng.integers(0, 2, T)
        r = (2 * rng.standard_normal(T)).astype(np.float32)
        d = {"none": np.zeros(T, bool), "all": np.ones(T, bool), "last": np.arange(T) == T - 1,
             "random": rng.random(T) < 0.1}[dones]
        alg.prepare_data(dict(cur_state=s, action=a, reward=r, next_state=s2, done=d))
        r64 = orc.nstep_returns(r, d, n, _f32(gamma))
        r32 = orc.nstep_returns(r, d, n, _f32(gamma), dtype=np.float32)
        refs.append(dict(r64=r64, r32=r32, s=s, s2=s2, a=a))
        sent += [(si, t) for t in range(T)]
    keep = sent[-cap:]
    assert len(sent) > cap and any(segs[si][0] < n for si, _ in keep)     # a wrap; a segment shorter than n in the ring
    b = alg.buff
    torch.cuda.synchronize()
    assert b.count == cap and b.head == len(sent) % cap
    slots = np.array([(len(sent) - cap + j) % cap for j in range(cap)])
    got = {k: getattr(b, k)[:cap].cpu().numpy() for k in ("obs", "action", "reward", "next_obs", "done", "disc")}
    want = {k: [] for k in ("obs", "action", "next_obs", "done", "r64", "d64", "r32", "d32")}
    for si, t in keep:
        f = refs[si]
        (r64, d64, last, dn), (r32, d32, _, _) = f["r64"], f["r32"]
        want["obs"].append(f["s"][t]); want["action"].append(f["a"][t]); want["next_obs"].append(f["s2"][last[t]])
        want["done"].append(dn[t]); want["r64"].append(r64[t]); want["d64"].append(d64[t])
        want["r32"].append(r32[t]); want["d32"].append(d32[t])
    want = {k: np.array(v) for k, v in want.items()}
    np.testing.assert_array_equal(got["obs"][slots], want["obs"])
    np.testing.assert_array_equal(got["action"][slots], want["action"])
    np.testing.assert_array_equal(got["next_obs"][slots], want["next_obs"])
    np.testing.assert_array_equal(got["done"][slots], want["done"].astype(np.uint8))
    assert want["done"].any() and not want["done"].all()
    bad = _within("dqn_nstep_ring/%s" % name, {"reward": (rel_err(got["reward"][slots], want["r64"]), rel_err(want["r32"], want["r64"])),
                                                "disc": (rel_err(got["disc"][slots], want["d64"]), rel_err(want["d32"], want["d64"]))})
    assert not bad, bad
