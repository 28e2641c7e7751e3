"""MuzeroMlp / MuzeroCnn on the H100 against the float64 oracle (tests/muzero_oracle.py): the training step (loss, every
weight gradient, a three-step loss trace) on both kernel paths and across support widths up to the kernel limit, the
batched and batch-1 inference, graph replay against eager launches, the input gradient of the backward pass, argument
checks that launch nothing, and the weight-list save/load round trip."""
import ctypes as C

import numpy as np
import pytest
import torch

import muzero_oracle as mo

pytestmark = pytest.mark.gpu


def _vmax_for_support(S):
    lo, hi = 0.0, 1e7
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if mo.support_size(0, mid) < S:
            lo = mid
        else:
            hi = mid
    assert mo.support_size(0, hi) == S
    return hi


def _model(name, state_dim, A, cfg, seed=0, graph=True):
    from xingtian_b200.registry import Registers
    torch.cuda.set_device(0)
    mc = dict(cfg, init_seed=seed, use_cuda_graph=graph)
    return Registers.model[name]({"model_name": name, "state_dim": list(state_dim), "action_dim": A, "model_config": mc})


def _archs(m):
    return (m.rep.arch, m.dyn.arch, m.pred.arch)


def _batch(rng, m, B, obs_shape, obs_u8):
    K, A = m.td_step, m.action_dim
    obs = rng.integers(0, 256, (B,) + obs_shape).astype(np.uint8) if obs_u8 else rng.normal(size=(B,) + obs_shape).astype(np.float32)
    if not obs_u8 and len(obs_shape) == 3:
        obs = rng.integers(0, 256, (B,) + obs_shape).astype(np.float32)
    action = rng.integers(0, A, (B, K)).astype(np.int32)
    tv = rng.uniform(m.value_min - 1, m.value_max + 1, (B, K + 1))
    tr = rng.uniform(m.reward_min - 0.5, m.reward_max + 0.5, (B, K + 1))
    tp = rng.dirichlet(np.ones(A), (B, K + 1))
    return obs, action, tv, tr, tp


def _check_step(m, B, obs_shape, obs_u8, steps, seed=0, rel=2e-3):
    rng = np.random.default_rng(seed)
    ref = mo.Learner(_archs(m), m.get_weights(), m.td_step, (m.value_min, m.value_max), (m.reward_min, m.reward_max), lr=m.learning_rate)
    for s in range(steps):
        obs, action, tv, tr, tp = _batch(rng, m, B, obs_shape, obs_u8)
        loss = m.train([obs, action, np.ones((B, 1))], [tv, tr, tp])
        rloss, rg = ref.train(obs, action, tv.astype(np.float32), tr.astype(np.float32), tp.astype(np.float32))
        assert abs(loss - rloss) <= rel * max(1.0, abs(rloss)), (s, loss, rloss)
        if s == 0:   # every weight gradient of the first step (rep / pred slices and the accumulated dynamics slice)
            g = m.grads.cpu().numpy()
            tables = m._tables()
            assert len(tables) == len(rg)
            for i, ((off, shape), r) in enumerate(zip(tables, rg)):
                r = r.numpy()
                d = g[off:off + r.size].reshape(r.shape)
                scale = max(float(np.abs(r).max()), 1e-6)
                assert float(np.abs(d - r).max()) <= rel * scale + 1e-7, (i, r.shape, float(np.abs(d - r).max()), scale)


@pytest.fixture(params=[1, 0], ids=["tc", "fp32"])
def tc_mode(request):
    from xingtian_b200 import capi
    lib = capi.lib()
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(request.param)
    yield request.param
    lib.xtb_set_tc_mode(old)


@pytest.mark.parametrize("S", [2, 8, 23, 305, 1024])
@pytest.mark.parametrize("B", [1, 37])
def test_mlp_train_vs_oracle_across_supports(S, B):
    vmax = 0.999 * _vmax_for_support(S + 1)   # well inside the range of values with support S
    m = _model("MuzeroMlp", (4,), 2, {"value_min": 0, "value_max": vmax, "reward_min": -2, "reward_max": 2, "max_batch": 64})
    assert m.value_support_size == S
    _check_step(m, B, (4,), False, 3)


def test_mlp_train_defaults_both_paths(tc_mode):
    m = _model("MuzeroMlp", (4,), 2, {"max_batch": 1024})
    assert sum(len(w.reshape(-1)) for w in m.get_weights()) == 23253 and (m.value_support_size, m.reward_support_size) == (305, 26)
    _check_step(m, 1024, (4,), False, 3)


def test_cnn_breakout_train_vs_oracle(tc_mode):
    cfg = {"reward_min": 0, "reward_max": 50, "value_min": 0, "value_max": 500, "obs_type": "uint8", "max_batch": 16}
    m = _model("MuzeroCnn", (84, 84, 4), 4, cfg)
    assert sum(w.size for w in m.get_weights()) == 1016355
    _check_step(m, 6, (84, 84, 4), True, 3)


def test_cnn_pong_shapes_float_frames(tc_mode):
    cfg = {"reward_min": -2, "reward_max": 2, "value_min": -21, "value_max": 21, "max_batch": 8}
    m = _model("MuzeroCnn", (84, 84, 4), 6, cfg)
    assert sum(w.size for w in m.get_weights()) == 1014416 and (m.value_support_size, m.reward_support_size) == (7, 3)
    _check_step(m, 3, (84, 84, 4), False, 1)


def test_inference_batched_and_batch1():
    cfg = {"reward_min": 0, "reward_max": 50, "value_min": 0, "value_max": 500, "obs_type": "uint8", "max_batch": 64}
    m = _model("MuzeroCnn", (84, 84, 4), 4, cfg, seed=3)
    archs, w = _archs(m), m.get_weights()
    rng = np.random.default_rng(5)
    obs = rng.integers(0, 256, (50, 84, 84, 4)).astype(np.uint8)
    rv, rp, rh = mo.initial_inference(archs, w, obs, (0, 500))
    ob = torch.from_numpy(obs).cuda()
    v, p, h = (t.cpu().numpy() for t in m.initial_inference_batch(ob, 50))
    np.testing.assert_allclose(h, rh, rtol=2e-3, atol=2e-3 * np.abs(rh).max())
    np.testing.assert_allclose(p, rp, atol=2e-4)
    np.testing.assert_allclose(v, rv, rtol=2e-3, atol=2e-3)
    np.testing.assert_allclose(m.value_inference(obs), rv, rtol=2e-3, atol=2e-3)
    act = rng.integers(0, 4, 50).astype(np.int32)
    sv, sr, sp, sh = mo.recurrent_inference(archs, w, h, act, (0, 500), (0, 50))
    v2, r2, p2, h2 = (t.cpu().numpy().copy() for t in m.recurrent_inference_batch(torch.from_numpy(h).cuda(), torch.from_numpy(act).cuda(), 50))
    np.testing.assert_allclose(h2, sh, rtol=2e-3, atol=2e-3 * np.abs(sh).max())
    np.testing.assert_allclose(p2, sp, atol=2e-4)
    np.testing.assert_allclose(v2, sv, rtol=2e-3, atol=2e-3)
    np.testing.assert_allclose(r2, sr, rtol=2e-3, atol=2e-3)
    # the batch-1 reference surface returns sample 0
    o = m.initial_inference(obs[:1])
    assert abs(o.value - v[0]) < 1e-4 * max(1, abs(v[0])) and o.reward == 0
    np.testing.assert_allclose(o.policy, p[0], atol=1e-6)
    o2 = m.recurrent_inference(h[0], int(act[0]))
    assert abs(o2.value - v2[0]) < 1e-4 * max(1, abs(v2[0])) and abs(o2.reward - r2[0]) < 1e-4 * max(1, abs(r2[0]))
    np.testing.assert_allclose(o2.hidden_state, h2[0], rtol=1e-5, atol=1e-6)


def test_graph_replay_matches_eager():
    """The captured step against the same launches issued eagerly.  The first layers of the dynamics and prediction nets
    read their float input on the fp32 kernels, whose split-K weight gradient sums with atomics: the two runs agree to
    float rounding, not bitwise."""
    from xingtian_b200 import capi
    cfg = {"reward_min": 0, "reward_max": 50, "value_min": 0, "value_max": 500, "obs_type": "uint8", "max_batch": 32}
    ms = [_model("MuzeroCnn", (84, 84, 4), 4, cfg, seed=7, graph=g) for g in (True, False)]
    rng = np.random.default_rng(9)
    batches = [_batch(rng, ms[0], 32, (84, 84, 4), True) for _ in range(3)]
    r0 = capi.lib().xtb_graph_replay_count()
    losses = [[m.train([b[0], b[1], None], list(b[2:])) for b in batches] for m in ms]
    assert capi.lib().xtb_graph_replay_count() - r0 == 3
    np.testing.assert_allclose(losses[0], losses[1], rtol=1e-5)
    w0, w1 = ms[0].params.cpu().numpy(), ms[1].params.cpu().numpy()
    assert np.abs(w0 - w1).max() <= 1e-5


def test_train_returns_post_update_values():
    m = _model("MuzeroMlp", (4,), 2, {"max_batch": 64, "value_min": -10, "value_max": 10})
    rng = np.random.default_rng(1)
    obs, action, tv, tr, tp = _batch(rng, m, 40, (4,), False)
    b = m._buffers(40)
    for k, a, dt in (("obs", obs, np.float32), ("action", action, np.int32), ("tv", tv, np.float32), ("tr", tr, np.float32),
                     ("tp", tp, np.float32)):
        b[k].copy_(torch.from_numpy(np.asarray(a, dt)))
    vals = torch.empty(40, device="cuda")
    m.train_device(b["obs"], b["action"], b["tv"], b["tr"], b["tp"], 40, b["loss"], vals)
    ref, _, _ = mo.initial_inference(_archs(m), m.get_weights(), obs, (-10, 10))
    np.testing.assert_allclose(vals.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)


def test_backward_input_gradient():
    from xingtian_b200.engine import Net
    torch.cuda.set_device(0)
    arch = dict(input_dtype="float32", state_dim=(40,), scale=1.0, layers=[
        ("a", "dense", "obs", dict(n=64, act="relu")), ("b", "dense", "a", dict(n=32, act="relu")),
        ("c", "dense", "obs", dict(n=32, act=None)), ("d", "dense", "b", dict(n=5, act=None))])
    net = Net(arch, max_batch=64)
    rng = np.random.default_rng(0)
    net.params.copy_(torch.from_numpy(rng.normal(0, 0.3, net.n_params).astype(np.float32)))
    net.params_changed()
    x = rng.normal(size=(33, 40)).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    net.forward(xd, 33)
    gd, gc = rng.normal(size=(33, 5)), rng.normal(size=(33, 32))
    net.tensor_grad("d")[:33].copy_(torch.from_numpy(gd.astype(np.float32)))
    net.tensor_grad("c")[:33].copy_(torch.from_numpy(gc.astype(np.float32)))
    dobs = torch.full((33, 40), float("nan"), device="cuda")
    net.backward_input(xd, 33, ["d", "c"], dobs)
    W = {k: torch.tensor(v.astype(np.float64)) for k, v in net.get_weights().items()}
    xt = torch.tensor(x.astype(np.float64), requires_grad=True)
    a = torch.relu(xt @ W["a/kernel"] + W["a/bias"])
    b = torch.relu(a @ W["b/kernel"] + W["b/bias"])
    c = xt @ W["c/kernel"] + W["c/bias"]
    d = b @ W["d/kernel"] + W["d/bias"]
    ((d * torch.tensor(gd)).sum() + (c * torch.tensor(gc)).sum()).backward()
    ref = xt.grad.numpy()
    np.testing.assert_allclose(dobs.cpu().numpy(), ref, rtol=1e-4, atol=1e-4 * np.abs(ref).max())


def test_invalid_arguments_launch_nothing():
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = capi.lib()
    m = _model("MuzeroMlp", (4,), 2, {"max_batch": 16})
    b = m._buffers(16)
    loss = b["loss"]

    def call(n, unroll=m.td_step):
        bt = capi.MuzeroBatch()
        bt.obs, bt.action, bt.target_value = b["obs"].data_ptr(), b["action"].data_ptr(), b["tv"].data_ptr()
        bt.target_reward, bt.target_policy, bt.unroll = b["tr"].data_ptr(), b["tp"].data_ptr(), unroll
        return lib.xtb_muzero_train(m.handle, m.opt.handle, C.byref(bt), n, 0.0, _ptr(loss), None, 1, stream_ptr())

    torch.cuda.synchronize()
    n0 = lib.xtb_launch_count()
    assert call(17) == -1                        # above max_batch
    assert call(0) == -1
    assert call(8, unroll=m.td_step + 1) == -1   # unroll mismatch
    assert lib.xtb_muzero_initial_inference(m.handle, None, 4, None, None, None, 1, stream_ptr()) == -1
    assert lib.xtb_muzero_recurrent_inference(m.handle, _ptr(b["hid_in"]), _ptr(b["act1"]), 17, None, None, None, None, 1,
                                              stream_ptr()) == -1
    hook = capi.GRAD_HOOK(lambda u, g, c, s: 1)
    lib.xtb_set_grad_hook(hook, None)
    try:
        assert call(8) == -3
    finally:
        lib.xtb_set_grad_hook(C.cast(None, capi.GRAD_HOOK), None)
    # the create-time checks: a support wider than the kernels take, nets not bound to one buffer
    desc = capi.MuzeroDesc(m.td_step, 2, 2, 3, 2, 3, 0.0, 10.0, 0.0, 10.0)
    out = C.c_void_p()
    assert lib.xtb_muzero_create(m.rep.handle, m.dyn.handle, m.pred.handle, C.byref(desc), 16, C.byref(out)) == 0
    lib.xtb_muzero_destroy(out)
    assert lib.xtb_muzero_create(m.pred.handle, m.dyn.handle, m.rep.handle, C.byref(desc), 16, C.byref(out)) == -1
    assert lib.xtb_muzero_create(m.rep.handle, m.dyn.handle, m.pred.handle, C.byref(desc), 17, C.byref(out)) == -1
    torch.cuda.synchronize()
    assert lib.xtb_launch_count() == n0
    with pytest.raises(ValueError):
        m._check_batch(17)
    big = _vmax_for_support(1025)
    with pytest.raises(RuntimeError):
        _model("MuzeroMlp", (4,), 2, {"max_batch": 4, "value_max": big})


def test_save_load_round_trip(tmp_path):
    m = _model("MuzeroMlp", (4,), 3, {"max_batch": 8}, seed=1)
    m2 = _model("MuzeroMlp", (4,), 3, {"max_batch": 8}, seed=2)
    path = m.save_model(str(tmp_path / "actor_00001"))
    m2.load_model(path)
    for a, b in zip(m.get_weights(), m2.get_weights()):
        np.testing.assert_array_equal(a, b)
    obs = np.random.default_rng(0).normal(size=(5, 4)).astype(np.float32)
    np.testing.assert_array_equal(m.value_inference(obs), m2.value_inference(obs))


def test_mlp_widest_support_full_batch():
    """S = 1024 at B = 1024: the widest rows and the largest grids of the cross-entropy and ordered-sum kernels."""
    vmax = 0.999 * _vmax_for_support(1025)
    m = _model("MuzeroMlp", (4,), 2, {"value_min": 0, "value_max": vmax, "max_batch": 1024})
    assert m.value_support_size == 1024
    _check_step(m, 1024, (4,), False, 2)


def test_cnn_pong_int8_frames_both_paths(tc_mode):
    """obs_type int8 (muzero_pong.yaml): every byte b decodes as (b < 128 ? b : b - 256) / 255 in the space-to-depth
    decode (tensor-core path) and in the fp32 im2col loader."""
    cfg = {"reward_min": -2, "reward_max": 2, "value_min": -21, "value_max": 21, "obs_type": "int8", "max_batch": 8}
    m = _model("MuzeroCnn", (84, 84, 4), 6, cfg)
    assert m.rep.layer_plan(0)["s2d"]      # planned onto the decode; tc_mode 0 runs the fp32 loader instead
    _check_step(m, 5, (84, 84, 4), True, 2)
    obs = np.random.default_rng(3).integers(0, 256, (7, 84, 84, 4)).astype(np.uint8)
    rv, _, _ = mo.initial_inference(_archs(m), m.get_weights(), obs, (-21, 21))
    np.testing.assert_allclose(m.value_inference(obs), rv, rtol=2e-3, atol=2e-3)
    # the int8 values themselves are accepted too (same bytes)
    np.testing.assert_array_equal(m.value_inference(obs.view(np.int8)), m.value_inference(obs))


class _OracleActor(object):
    """the float64 model behind the oracle learner"""

    def __init__(self, m):
        self.archs, self.vr, self.rr = _archs(m), (m.value_min, m.value_max), (m.reward_min, m.reward_max)
        self.ref = mo.Learner(self.archs, m.get_weights(), m.td_step, self.vr, self.rr, lr=m.learning_rate)
        self.td_step = m.td_step

    def value_inference(self, s):
        return mo.initial_inference(self.archs, self.ref.weights(), np.asarray(s), self.vr)[0]

    def train_and_values(self, image, actions, tv, tr, tp):
        loss, _ = self.ref.train(image, actions, tv.astype(np.float32), tr.astype(np.float32), tp.astype(np.float32))
        return loss, self.value_inference(image)


def test_learner_against_oracle_learner():
    import random
    from xingtian_b200 import alg_builder
    from xingtian_b200.algorithm import muzero as mz
    info = {"actor": {"model_name": "MuzeroMlp", "state_dim": [4], "action_dim": 3,
                      "model_config": {"max_batch": 8, "init_seed": 5, "value_min": -5, "value_max": 5,
                                       "reward_min": -2, "reward_max": 2}}}
    alg = alg_builder("Muzero", info, {"instance_num": 1, "agent_num": 1, "BATCH_SIZE": 8, "BUFFER_SIZE": 12, "UNROLL_STEP": 5})
    ref = object.__new__(mz.Muzero)
    ref.actor, ref.buff, ref.unroll_step, ref.batch_size = _OracleActor(alg.actor), mz.PrioritizedBuffer(12, 1), 5, 8
    rng = np.random.default_rng(0)
    trajs = []
    for t in range(14):
        L = int(rng.integers(5, 16))
        trajs.append(dict(cur_state=rng.normal(size=(L, 4)).astype(np.float32), action=rng.integers(0, 3, L),
                          reward=rng.uniform(-2, 2, L), done=np.zeros(L, bool), root_value=rng.normal(size=L),
                          child_visits=rng.dirichlet(np.ones(3), L), target_value=rng.uniform(-5, 5, L), tid=t))
    for learner in (alg, ref):
        for tr in trajs:
            learner.prepare_data(dict(tr))
    np.testing.assert_allclose([alg.buff.it_sum[i] for i in range(len(alg.buff))],
                               [ref.buff.it_sum[i] for i in range(len(ref.buff))], rtol=1e-4, atol=1e-5)
    for step in range(3):
        draws = []
        for learner in (alg, ref):
            random.seed(100 + step)
            state = random.getstate()
            trajs_s, pos, *_ = learner.sample_batch()
            draws.append(([t["tid"] for t in trajs_s], pos))
            random.setstate(state)
            loss = learner.train()
            draws[-1] += (loss,)
        assert draws[0][:2] == draws[1][:2], (step, draws)
        assert abs(draws[0][2] - draws[1][2]) <= 2e-3 * max(1.0, abs(draws[1][2])), (step, draws)
        np.testing.assert_allclose([alg.buff.it_sum[i] for i in range(len(alg.buff))],
                                   [ref.buff.it_sum[i] for i in range(len(ref.buff))], rtol=2e-3, atol=1e-4)
    with pytest.raises(ValueError):
        alg_builder("Muzero", info, {"instance_num": 1, "agent_num": 1, "UNROLL_STEP": 4})
    mz.UNROLL_STEP = 5
