"""Prioritized replay on the device (xtb_per_*, xtb_dqn_train_weighted, xtb_dqn_per_train): the sum / min trees against
the float64 restatement in per_oracle, the stratified draw and its importance weights, the weighted TD step of DqnCnn /
DqnMlp against a float64 restatement of the oracle's DqnLearner with per-row weights (the bounds of test_gpu_dueling),
the alpha = 0 step against the uniform one, one graph while the ring fills, and the DQN plugin with prioritized_replay."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from per_oracle import PerTree, descend, weights
from test_gpu_dueling import _restore_dqn_config  # noqa: F401  (autouse: module config globals restored after each test)
from test_gpu_kernels import _keepalive, dev, l2_rel, one_rank_comm, xb  # noqa: F401
from test_gpu_plugins import alg_cfg

pytestmark = pytest.mark.gpu


class Per(object):
    """an xtb_per handle with host-side helpers"""

    def __init__(self, capacity, alpha, eps=1e-6, seed=0):
        from xingtian_b200 import capi
        self.lib, self.check = capi.lib(), capi.check
        h = C.c_void_p()
        self.check(self.lib.xtb_per_create(capacity, alpha, eps, seed, C.byref(h)))
        self.h = h

    def __del__(self):
        self.lib.xtb_per_destroy(self.h)

    def add(self, first, n):
        from xingtian_b200.engine import stream_ptr
        self.check(self.lib.xtb_per_add(self.h, first, n, stream_ptr()))

    def update(self, idx, td_abs):
        from xingtian_b200.engine import _ptr, stream_ptr
        self.check(self.lib.xtb_per_update(self.h, _ptr(dev(np.asarray(idx, np.int32))), _ptr(dev(np.asarray(td_abs, np.float32))),
                                           len(idx), stream_ptr()))

    def sample(self, B, beta, u=None):
        from xingtian_b200.engine import _ptr, stream_ptr
        idx = torch.empty(B, dtype=torch.int32, device="cuda")
        w = torch.empty(B, dtype=torch.float32, device="cuda")
        self.check(self.lib.xtb_per_sample(self.h, B, beta, _ptr(dev(np.asarray(u, np.float64)) if u is not None else None), _ptr(idx),
                                           _ptr(w), stream_ptr()))
        return idx.cpu().numpy(), w.cpu().numpy()

    def state(self):
        return per_state(self.h)


def per_state(h):
    """xtb_per_state of handle h: the trees (float64, heap order) and the device scalars"""
    from xingtian_b200 import capi
    lib = capi.lib()
    leaves, count, status, mp, off = C.c_int(), C.c_int(), C.c_int(), C.c_double(), C.c_ulonglong()
    capi.check(lib.xtb_per_state(h, C.byref(leaves), None, None, None, None, None, None))
    s, m = np.empty(2 * leaves.value), np.empty(2 * leaves.value)
    capi.check(lib.xtb_per_state(h, None, C.byref(count), C.byref(mp), C.byref(status), C.byref(off), s.ctypes.data,
                                 m.ctypes.data))
    return dict(leaves=leaves.value, count=count.value, max_priority=mp.value, status=status.value, offset=off.value, sum=s, mn=m)


def _assert_internal_nodes(st):
    L = st["leaves"]
    node = np.arange(1, L)
    assert np.array_equal(st["sum"][node], st["sum"][2 * node] + st["sum"][2 * node + 1])
    assert np.array_equal(st["mn"][node], np.minimum(st["mn"][2 * node], st["mn"][2 * node + 1]))


def _filled(capacity, alpha, seed, eps=1e-6):
    """a device tree and its restatement after inserts, updates with repeated indices (and differing values), and
    inserts past the end of the ring that wrap onto the oldest slots"""
    rng = np.random.default_rng(seed)
    per, ref = Per(capacity, alpha, eps, seed=seed), PerTree(capacity, alpha, eps)
    head = count = 0
    for step in range(12):
        n = int(rng.integers(1, capacity // 3 + 2))
        while n:
            k = min(n, capacity - head)
            per.add(head, k); ref.add(head, k)
            head = (head + k) % capacity; count = min(capacity, count + k); n -= k
        m = int(rng.integers(1, 3 * capacity))
        idx = rng.integers(0, count, m)
        idx[m // 2:] = idx[:m - m // 2]                          # every index of the second half repeats an earlier one
        td = (rng.exponential(1.0, m) * (10.0 if step == 5 else 1.0)).astype(np.float32)
        per.update(idx, td); ref.update(idx, td)
    return per, ref


@pytest.mark.parametrize("capacity", [1, 7, 100, 4096])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 0.6])
def test_tree_matches_float64(xb, capacity, alpha):
    per, ref = _filled(capacity, alpha, seed=capacity)
    st = per.state()
    _assert_internal_nodes(st)
    assert st["leaves"] == ref.leaves and st["count"] == ref.count and st["status"] == 0
    assert st["max_priority"] == ref.max_priority
    L = st["leaves"]
    if alpha in (0.0, 1.0):
        assert np.array_equal(st["sum"][L:], ref.sum[L:]) and np.array_equal(st["mn"][L:], ref.mn[L:])
    else:
        np.testing.assert_allclose(st["sum"][L:], ref.sum[L:], rtol=1e-12, atol=0)
        assert np.array_equal(st["sum"][L + ref.count:], np.zeros(L - ref.count))
        assert np.all(np.isinf(st["mn"][L + ref.count:]))


def test_update_last_writer_wins_and_nonfinite(xb):
    per = Per(8, 1.0, eps=0.5)
    per.add(0, 8)
    per.update([3, 5, 3, 5, 2], [1.5, 0.5, 2.5, np.nan, np.inf])    # 3: the later 3.0; 5: NaN skipped, 1.0 stays; 2: skipped
    st = per.state()
    assert list(st["sum"][8:]) == [1, 1, 1, 3, 1, 1, 1, 1] and st["max_priority"] == 3.0
    assert st["status"] == 1
    _assert_internal_nodes(st)


@pytest.mark.parametrize("capacity,seed,B", [(100, 100, 512), (4096, 3000, 512), (1000, 37, 1500), (1, 1, 5)])
def test_injected_draws_match_host_descent(xb, capacity, seed, B):
    per, _ = _filled(capacity, 0.6, seed=seed)
    st = per.state()
    u = np.random.default_rng(B).random(B)
    u[:3] = [0.0, 0.5, 1.0 - 2 ** -53]
    idx, w = per.sample(B, 0.4, u)
    L, count = st["leaves"], st["count"]
    ref_idx = descend(st["sum"], L, count, u)
    assert np.array_equal(idx, ref_idx)
    np.testing.assert_allclose(w, weights(st["sum"], st["mn"], L, count, ref_idx, 0.4), rtol=1e-6)
    assert per.state()["offset"] == 0                          # injected draws leave the Philox counter alone


def test_philox_draws_reproducible_and_proportional(xb):
    from scipy import stats
    cap = 64
    pri = np.random.default_rng(1).uniform(0.1, 2.0, cap).astype(np.float32)
    mk = lambda seed: Per(cap, 1.0, eps=1e-6, seed=seed)   # noqa: E731
    a, b, c = mk(7), mk(7), mk(8)
    for p in (a, b, c):
        p.add(0, cap)
        p.update(np.arange(cap), pri)
    first = [a.sample(1000, 0.4) for _ in range(3)]
    again = [b.sample(1000, 0.4) for _ in range(3)]
    for (i1, w1), (i2, w2) in zip(first, again):
        assert np.array_equal(i1, i2) and np.array_equal(w1, w2)
    assert not np.array_equal(first[0][0], first[1][0])      # the offset advanced
    assert not np.array_equal(c.sample(1000, 0.4)[0], first[0][0])
    assert a.state()["offset"] == 3
    counts = np.bincount(np.concatenate([i for i, _ in first] + [a.sample(1000, 0.4)[0] for _ in range(297)]), minlength=cap)
    st = a.state()
    leaf = st["sum"][st["leaves"]:]
    expect = leaf / leaf.sum() * counts.sum()
    assert counts.sum() == 300000
    assert stats.chisquare(counts, expect).pvalue > 1e-3


# ------------------------------------------------------------------------------------------- the weighted step
def _models(kind, A, dueling, seed=9):
    from xingtian_b200.model.dqn import DqnCnn, DqnMlp
    cls, sd = (DqnCnn, [84, 84, 4]) if kind == "cnn" else (DqnMlp, [4])
    mk = lambda: cls({"state_dim": sd, "action_dim": A, "model_config": {"dueling": dueling, "init_seed": seed, "LR": 0.00015}})  # noqa: E731
    return mk(), mk()


def _transitions(kind, n, A, seed):
    rng = np.random.default_rng(seed)
    if kind == "cnn":
        s = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8); s2 = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)
    else:
        s = rng.standard_normal((n, 4)).astype(np.float32); s2 = rng.standard_normal((n, 4)).astype(np.float32)
    return s, rng.integers(0, A, n).astype(np.int32), rng.standard_normal(n).astype(np.float32), s2, rng.random(n) < 0.1


def _weighted_reference(arch, w0, batch, wts, clipnorm, double, huber, disc):
    """DqnLearner's step (oracle) in float64 with the per-row weights of Keras sample_weight: loss = mean over B*A of
    w_b e_ba; returns the loss, |y - Q(s, a)| and the updated weights"""
    s, a, r, s2, d = batch
    with orc.precision("f64"):
        ref = orc.DqnLearner(arch, w0, lr=0.00015, clipnorm=clipnorm, double_dqn=double)
        y = orc.dqn_targets(ref.predict(s), ref.predict(s2, target=True), a, r, d, ref.gamma,
                            ref.predict(s2) if double else None, disc)
        q = orc.forward(ref.arch, ref.named(), s)[0]
        diff = q - torch.from_numpy(np.asarray(y)).to(q.dtype)
        if huber > 0:
            ad = diff.abs()
            per = torch.where(ad <= huber, 0.5 * diff * diff, huber * (ad - 0.5 * huber))
        else:
            per = diff * diff
        loss = (per * torch.from_numpy(wts.astype(np.float64))[:, None]).mean()
        grads = torch.autograd.grad(loss, ref.params)
        if clipnorm:
            grads = orc.clip_per_tensor(grads, clipnorm)
        ref.opt.step(grads)
        td = np.abs(diff.detach().numpy()[np.arange(len(a)), a.astype(np.int64)])
        return float(loss.detach()), td, ref.weights()


VARIANTS = {"plain": {}, "double": dict(double=True), "dueling": dict(dueling=True),
            "dueling_layers": dict(dueling=True, fuse=False), "huber": dict(huber=1.0), "nstep": dict(nstep=True),
            "dueling_double_nstep_huber": dict(dueling=True, double=True, nstep=True, huber=1.0)}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("kind", ["cnn", "mlp"])
def test_weighted_step_matches_float64(xb, kind, variant):
    from xingtian_b200 import capi
    v = VARIANTS[variant]
    dueling, double, huber, fuse = v.get("dueling", False), v.get("double", False), v.get("huber", 0.0), v.get("fuse", True)
    A, B, ring = 4, 32, 48
    model, tgt = _models(kind, A, dueling)
    w0 = model.get_weights()
    s, a, r, s2, d = _transitions(kind, ring, A, seed=3)
    rng = np.random.default_rng(5)
    idx = rng.integers(0, ring, B).astype(np.int32)
    idx[-4:] = idx[:4]                                       # repeated rows, as a draw with replacement gives
    wts = rng.uniform(0.1, 1.0, B).astype(np.float32)
    disc = np.where(d, 0.0, 0.99 ** 3).astype(np.float32) if v.get("nstep") else None
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    td = torch.zeros(B, dtype=torch.float32, device="cuda")
    capi.lib().xtb_set_fuse_heads(1 if fuse else 0)
    try:
        model.train_td_device(tgt, dev(s), dev(a), dev(r), dev(s2), dev(d.astype(np.uint8)), B, 0.99, loss, double_dqn=double,
                              idx=dev(idx), disc=dev(disc) if disc is not None else None, huber_delta=huber, weights=dev(wts), td_abs=td)
        got, got_td = float(loss.cpu()[0]), td.cpu().numpy()
    finally:
        capi.lib().xtb_set_fuse_heads(1)
    arch = model.arch
    want, want_td, rw = _weighted_reference(arch, w0, (s[idx], a[idx], r[idx], s2[idx], d[idx]), wts,
                                            10.0 if kind == "cnn" else None, double, huber, disc[idx] if disc is not None else None)
    assert abs(got - want) < 5e-3 * max(1.0, abs(want)), (got, want)
    assert np.max(np.abs(got_td - want_td)) < 5e-3 * max(1.0, float(np.max(want_td))), (got_td, want_td)
    w1 = model.get_weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0]); rupd = np.concatenate([(rw[k] - w0[k]).ravel() for k in w0])
    assert l2_rel(upd, rupd) < 5e-2


def _per_step_buffers(B):
    z = lambda dt: torch.zeros(B, dtype=dt, device="cuda")   # noqa: E731
    return dict(idx=z(torch.int32), w=z(torch.float32), td=z(torch.float32), status=torch.zeros(1, dtype=torch.int32, device="cuda"),
                loss=torch.zeros(1, dtype=torch.float32, device="cuda"))


@pytest.mark.parametrize("kind,dueling", [("cnn", True), ("cnn", False), ("mlp", False)])
def test_alpha_zero_step_is_the_uniform_step(xb, kind, dueling):
    """alpha = 0 makes every priority 1 and every weight exactly 1: the prioritized graph on its own draw gives the uniform
    step on the same rows bit for bit"""
    A, B, ring = 4, 32, 96
    m_per, tgt = _models(kind, A, dueling)
    m_uni, _ = _models(kind, A, dueling)
    s, a, r, s2, d = [dev(x) for x in _transitions(kind, ring, A, seed=8)]
    d = d.to(torch.uint8)
    per = Per(ring, 0.0, seed=4)
    per.add(0, ring)
    b = _per_step_buffers(B)
    m_per.train_per_device(tgt, per.h, 0.4, s, a, r, s2, d, B, 0.99, b["loss"], b["idx"], b["w"], b["td"], b["status"])
    assert torch.all(b["w"] == 1.0) and int(b["status"].cpu()[0]) == 0
    loss_uni = torch.zeros(1, dtype=torch.float32, device="cuda")
    m_uni.train_td_device(tgt, s, a, r, s2, d, B, 0.99, loss_uni, idx=b["idx"].clone())
    assert torch.equal(m_per.net.params, m_uni.net.params)
    lp, lu = float(b["loss"].cpu()[0]), float(loss_uni.cpu()[0])
    assert abs(lp - lu) <= 1e-6 * max(1.0, abs(lu)), (lp, lu)
    st = per.state()
    assert st["offset"] == 1 and np.all(st["sum"][st["leaves"]:st["leaves"] + ring] == 1.0)


def test_one_graph_while_the_ring_fills(xb):
    """count, max_priority and the Philox offset are read on the device: one capture serves every step"""
    from xingtian_b200 import capi
    lib = capi.lib()
    A, B, ring = 3, 16, 64
    model, tgt = _models("mlp", A, False)
    s, a, r, s2, d = [dev(x) for x in _transitions("mlp", ring, A, seed=2)]
    d = d.to(torch.uint8)
    per = Per(ring, 0.6, seed=1)
    b = _per_step_buffers(B)
    per.add(0, 5)
    torch.cuda.synchronize()
    caps, reps = lib.xtb_graph_capture_count(), lib.xtb_graph_replay_count()
    head, count, steps = 5, 5, 0
    for _ in range(20):
        model.train_per_device(tgt, per.h, 0.4, s, a, r, s2, d, B, 0.99, b["loss"], b["idx"], b["w"], b["td"], b["status"])
        steps += 1
        assert 0 <= int(b["idx"].cpu().min()) and int(b["idx"].cpu().max()) < count
        k = min(7, ring - head)
        per.add(head, k)
        head, count = (head + k) % ring, min(ring, count + k)
    torch.cuda.synchronize()
    assert lib.xtb_graph_capture_count() - caps == 1
    assert lib.xtb_graph_replay_count() - reps == steps
    st = per.state()
    assert st["count"] == ring and st["offset"] == steps and st["status"] == 0 and st["max_priority"] > 1.0
    _assert_internal_nodes(st)


# ------------------------------------------------------------------------------------------- the DQN plugin
def _plugin(kind, **kw):
    import xingtian_b200 as xb_
    if kind == "cnn":
        info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": 4, "model_config": {"init_seed": 3}}}
    else:
        info = {"actor": {"model_name": "DqnMlp", "state_dim": [4], "action_dim": 2, "model_config": {"init_seed": 3}}}
    cfg = dict(BUFFER_SIZE=200, BATCH_SIZE=32, TARGET_UPDATE_FREQ=2, prioritized_replay=True, PRIORITY_ALPHA=0.6, priority_beta=0.5)
    cfg.update(kw)
    return xb_.alg_builder("DQN", info, alg_cfg(**cfg))


def _segment(alg, T, seed):
    rng = np.random.default_rng(seed)
    A = alg.actor.action_dim
    sd = tuple(alg.actor.state_dim)
    if len(sd) == 3:
        s = rng.integers(0, 256, (T + 1,) + sd, dtype=np.uint8)
    else:
        s = rng.standard_normal((T + 1,) + sd).astype(np.float32)
    return dict(cur_state=s[:-1], action=rng.integers(0, A, T), reward=rng.standard_normal(T).astype(np.float32),
                next_state=s[1:], done=rng.random(T) < 0.05)


def _assert_priorities_refreshed(alg):
    """the leaves of the last step's rows hold (|delta| + eps) ** alpha of the last draw naming them"""
    st = per_state(alg.buff.per)
    idx, td = alg._per_idx.cpu().numpy(), alg._per_td.cpu().numpy()
    last = {int(j): k for k, j in enumerate(idx)}
    for j, k in last.items():
        want = (float(td[k]) + 1e-6) ** 0.6
        assert abs(st["sum"][st["leaves"] + j] - want) <= 1e-12 * want, (j, st["sum"][st["leaves"] + j], want)
    assert st["max_priority"] >= max(float(t) + 1e-6 for t in td)
    _assert_internal_nodes(st)


@pytest.mark.parametrize("kind,n_step", [("cnn", 1), ("mlp", 1), ("mlp", 3), ("cnn", 3)])
def test_plugin_prioritized_train(xb, kind, n_step):
    alg = _plugin(kind, N_STEP=n_step)
    assert alg.prioritized and alg.n_step == n_step and alg.priority_beta == 0.5
    w0 = alg.get_weights()
    from xingtian_b200 import capi
    caps = capi.lib().xtb_graph_capture_count()
    for i in range(4):
        alg.prepare_data(_segment(alg, 60, seed=i))               # 240 rows into a 200-slot ring: it wraps
        loss = alg.train()
        assert np.isfinite(loss)
        _assert_priorities_refreshed(alg)
    assert alg.buff.count == 200 and alg.train_count == 4
    assert capi.lib().xtb_graph_capture_count() - caps == 1
    assert list(alg.get_weights()) == list(w0)
    assert any(not np.array_equal(alg.get_weights()[k], w0[k]) for k in w0)


def test_plugin_raises_on_nonfinite_priority(xb):
    from xingtian_b200.engine import _ptr, stream_ptr
    alg = _plugin("mlp")
    alg.prepare_data(_segment(alg, 50, seed=1))
    assert np.isfinite(alg.train())
    lib = alg.actor.net.lib
    assert lib.xtb_per_update(alg.buff.per, _ptr(dev(np.array([3], np.int32))), _ptr(dev(np.array([np.nan], np.float32))), 1,
                              stream_ptr()) == 0
    with pytest.raises(FloatingPointError):
        alg.train()


def test_uniform_plugin_has_no_tree(xb):
    alg = _plugin("mlp", prioritized_replay=False)
    assert alg.buff.per is None and not alg.prioritized
    alg.prepare_data(_segment(alg, 50, seed=1))
    assert np.isfinite(alg.train())


def test_invalid_arguments(xb):
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = capi.lib()
    h = C.c_void_p()
    for cap, alpha, eps in ((0, 0.6, 1e-6), (-3, 0.6, 1e-6), (8, -0.1, 1e-6), (8, float("nan"), 1e-6), (8, 0.6, 0.0),
                            (8, 0.6, -1.0), (8, 0.6, float("inf"))):
        assert lib.xtb_per_create(cap, alpha, eps, 0, C.byref(h)) == -1 and not h.value, (cap, alpha, eps)
    assert lib.xtb_per_create(8, 0.6, 1e-6, 0, None) == -1
    per = Per(8, 0.6)
    per.add(0, 8)
    i = torch.zeros(4, dtype=torch.int32, device="cuda"); w = torch.zeros(4, dtype=torch.float32, device="cuda")
    model, tgt = _models("mlp", 2, False)
    model._td_scratch(tgt, 4)
    b = _per_step_buffers(4)
    obs = torch.zeros(8, 4, device="cuda"); act = torch.zeros(8, dtype=torch.int32, device="cuda")
    rew = torch.zeros(8, device="cuda"); don = torch.zeros(8, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    n0 = lib.xtb_launch_count()
    s = stream_ptr()
    assert lib.xtb_per_add(per.h, 6, 3, s) == -1 and lib.xtb_per_add(per.h, -1, 2, s) == -1 and lib.xtb_per_add(per.h, 0, 0, s) == -1
    assert lib.xtb_per_add(None, 0, 1, s) == -1
    for B, beta in ((0, 0.4), (-2, 0.4), (4, 0.0), (4, -1.0), (4, float("nan"))):
        assert lib.xtb_per_sample(per.h, B, beta, None, _ptr(i), _ptr(w), s) == -1, (B, beta)
    assert lib.xtb_per_sample(per.h, 4, 0.4, None, None, _ptr(w), s) == -1
    assert lib.xtb_per_update(per.h, _ptr(i), _ptr(w), 0, s) == -1 and lib.xtb_per_update(per.h, None, _ptr(w), 4, s) == -1
    for beta, n in ((0.0, 4), (float("inf"), 4)):
        with pytest.raises(RuntimeError, match="beta"):
            model.train_per_device(tgt, per.h, beta, obs, act, rew, obs, don, n, 0.99, b["loss"], b["idx"], b["w"], b["td"], b["status"])
    assert lib.xtb_launch_count() == n0
    with one_rank_comm():
        assert lib.xtb_per_add(per.h, 0, 1, s) == -3 and b"data-parallel" in lib.xtb_last_error()
        assert lib.xtb_per_sample(per.h, 4, 0.4, None, _ptr(i), _ptr(w), s) == -3
        assert lib.xtb_per_update(per.h, _ptr(i), _ptr(w), 4, s) == -3
        with pytest.raises(RuntimeError, match="data-parallel"):
            model.train_per_device(tgt, per.h, 0.4, obs, act, rew, obs, don, 4, 0.99, b["loss"], b["idx"], b["w"], b["td"], b["status"])
    assert lib.xtb_launch_count() == n0
