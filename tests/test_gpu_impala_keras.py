"""IMPALA with ImpalaMlp / ImpalaCnn on the device against the float64 oracle (tests/impala_keras_oracle.py): the V-trace
variant of the train entry point, the Keras fit epoch on both kernel paths, IMPALA end to end, Adam `decay`, CUDA-graph
replay, argument validation and weight I/O.

Bounds are those of test_gpu_dueling: loss within 5e-3 relative, the weight update within 5e-2 L2-relative of the float64
oracle's (it absorbs a ReLU that flips between fp32 and float64 near zero)."""
import ctypes as C

import numpy as np
import pytest
import torch

import impala_keras_oracle as iko
from oracle import xt_oracle as orc
from test_gpu_kernels import _keepalive, dev, l2_rel, rel_err, xb  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_config():
    """import_config writes configs into module globals, as the reference does: restore them after every test"""
    from xingtian_b200.algorithm import impala as alg_mod
    from xingtian_b200.model import impala_cnn, impala_mlp
    saved = [(m, {k: v for k, v in vars(m).items() if k.isupper()}) for m in (alg_mod, impala_cnn, impala_mlp)]
    yield
    for m, d in saved:
        for k, v in d.items():
            setattr(m, k, v)


def _mlp(A=2, seed=1, **cfg):
    from xingtian_b200.model.impala_mlp import ImpalaMlp
    return ImpalaMlp({"state_dim": [4], "action_dim": A, "model_config": dict(init_seed=seed, **cfg)})


def _cnn(A=4, seed=2, **cfg):
    from xingtian_b200.model.impala_cnn import ImpalaCnn
    return ImpalaCnn({"state_dim": [84, 84, 4], "action_dim": A, "model_config": dict(init_seed=seed, **cfg)})


def _alg(model_name, A, L, batch, state_dim, seed=3, **mcfg):
    import xingtian_b200 as xb_
    info = {"actor": {"model_name": model_name, "state_dim": state_dim, "action_dim": A,
                      "model_config": dict(init_seed=seed, **mcfg)}}
    return xb_.alg_builder("IMPALA", info, {"instance_num": 2, "agent_num": 1, "BATCH_SIZE": batch, "episode_len": L})


def _trajs(n, L, A, state_dim, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        shape = (L + 1,) + tuple(state_dim)
        s = rng.integers(0, 256, shape, dtype=np.uint8) if len(state_dim) == 3 else rng.standard_normal(shape).astype(np.float32)
        lg = rng.standard_normal((L, A)).astype(np.float32)
        bp = np.exp(lg) / np.exp(lg).sum(-1, keepdims=True)
        out.append(dict(cur_state=s, real_action=np.eye(A)[rng.integers(0, A, L)], action=bp.astype(np.float32),
                        reward=[float(x) for x in rng.choice([-1.0, 0.0, 1.0], size=L)],
                        done=[bool(x) for x in rng.random(L) < 0.05]))
    return out


def _upd(w1, w0):
    return np.concatenate([(w1[k] - w0[k]).ravel() for k in w0])


# ------------------------------------------------------------------------------------------- V-trace
@pytest.mark.parametrize("A", [2, 4, 18])
@pytest.mark.parametrize("L", [1, 31, 33, 200])
@pytest.mark.parametrize("n_traj", [1, 3])
def test_vtrace_matches_float64(xb, n_traj, L, A):
    """pg_adv / target value of the train entry against the float64 variant on the pre-update weights"""
    alg = _alg("ImpalaMlp", A, L, 512, [4])
    trajs = _trajs(n_traj, L, A, (4,), seed=L + A)
    w0 = alg.get_weights()
    for tr in trajs:
        alg.prepare_data(tr)
    alg.train()
    pg, tv = alg.pg_adv.cpu().numpy(), alg.target_value.cpu().numpy()
    with orc.precision("f64"):
        ref = iko.ImpalaKerasLearner(iko.impala_mlp_arch(action_dim=A), w0)
        probs, values = ref.predict(np.concatenate([t["cur_state"] for t in trajs]))
    st = lambda k: np.stack([np.asarray(t[k]) for t in trajs])   # noqa: E731
    rpg, rtv = iko.vtrace(probs.reshape(n_traj, L + 1, A), values.reshape(n_traj, L + 1), st("action"), st("real_action"),
                          st("reward"), st("done"))
    assert rel_err(pg, rpg) < 1e-4, rel_err(pg, rpg)
    assert rel_err(tv, rtv) < 1e-4, rel_err(tv, rtv)


# ------------------------------------------------------------------------------------------- one fit epoch
def _fit_case(model, arch, n, seed, clipnorm, decay=0.0, lr=3e-4):
    rng = np.random.default_rng(seed)
    shape = (n,) + tuple(arch["state_dim"])
    obs = rng.integers(0, 256, shape, dtype=np.uint8) if arch["input_dtype"] == "uint8" else rng.standard_normal(shape).astype(np.float32)
    A = model.action_dim
    y = np.eye(A, dtype=np.float32)[rng.integers(0, A, n)]
    adv, tv = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    w0 = model.get_weights()
    np.random.seed(seed)
    loss = model.train([obs, adv[:, None]], [y, tv[:, None]])
    with orc.precision("f64"):
        ref = iko.ImpalaKerasLearner(arch, w0, lr=lr, clipnorm=clipnorm, decay=decay)
        np.random.seed(seed)
        rloss = ref.fit(obs, adv, y, tv)
        rw = ref.weights()
    return loss, rloss, w0, model.get_weights(), rw


@pytest.mark.parametrize("tc", [1, 0])
@pytest.mark.parametrize("kind,A", [("mlp", 2), ("cnn", 4), ("cnn", 18)])
def test_fit_matches_oracle(xb, tc, kind, A):
    """model.train: 300 rows = minibatches 128 / 128 / 44, on both kernel paths"""
    lib = xb["lib"]
    lib.xtb_set_tc_mode(tc)
    try:
        model = _mlp(A) if kind == "mlp" else _cnn(A)
        arch = iko.impala_mlp_arch(action_dim=A) if kind == "mlp" else iko.impala_cnn_arch(action_dim=A)
        assert list(model.get_weights()) == list(orc.param_shapes(arch))
        torch.cuda.synchronize()
        n0 = lib.xtb_launch_count()
        loss, rloss, w0, w1, rw = _fit_case(model, arch, 300, 7, None if kind == "mlp" else 40.0)
        assert lib.xtb_launch_count() > n0
    finally:
        lib.xtb_set_tc_mode(1)
    assert abs(loss - rloss) < 5e-3 * max(1.0, abs(rloss)), (loss, rloss)
    assert l2_rel(_upd(w1, w0), _upd(rw, w0)) < 5e-2


def test_adam_decay_matches_oracle(xb):
    """an exaggerated decay (0.1) over 5 Adam steps (640 rows), and not the undecayed result"""
    model = _mlp(4, LR=0.01)
    model.opt.set_decay(0.1)
    arch = iko.impala_mlp_arch(action_dim=4)
    loss, rloss, w0, w1, rw = _fit_case(model, arch, 640, 9, None, decay=0.1, lr=0.01)
    assert abs(loss - rloss) < 5e-3 * max(1.0, abs(rloss)), (loss, rloss)
    err = l2_rel(_upd(w1, w0), _upd(rw, w0))
    assert err < 5e-3, err
    with orc.precision("f64"):
        plain = iko.ImpalaKerasLearner(arch, w0, lr=0.01)
        np.random.seed(9)
        rng = np.random.default_rng(9)
        obs = rng.standard_normal((640, 4)).astype(np.float32)
        y = np.eye(4, dtype=np.float32)[rng.integers(0, 4, 640)]
        adv, tv = rng.standard_normal(640).astype(np.float32), rng.standard_normal(640).astype(np.float32)
        plain.fit(obs, adv, y, tv)
    assert l2_rel(_upd(w1, w0), _upd(plain.weights(), w0)) > 10 * err


# ------------------------------------------------------------------------------------------- IMPALA end to end
def _run_alg(alg, arch, trajs_per_call, L, A, state_dim, batch, calls=3, clipnorm=None, decay=0.0):
    w0 = alg.get_weights()
    with orc.precision("f64"):
        ref = iko.ImpalaKerasLearner(arch, w0, clipnorm=clipnorm, decay=decay, batch_size=batch)
    for c in range(calls):
        trajs = _trajs(trajs_per_call, L, A, state_dim, seed=100 + c)
        for tr in trajs:
            alg.prepare_data(tr)
        np.random.seed(c)
        loss = alg.train()
        with orc.precision("f64"):
            np.random.seed(c)
            rloss, _ = ref.train(trajs)
        assert abs(loss - rloss) < 5e-3 * max(1.0, abs(rloss)), (c, loss, rloss)
        assert rel_err(alg.pg_adv.cpu().numpy(), ref.last["pg_adv"]) < 2e-3
    assert l2_rel(_upd(alg.get_weights(), w0), _upd(ref.weights(), w0)) < 5e-2
    return alg


def test_impala_cartpole_config_matches_oracle(xb):
    """examples/cartpole_impala.yaml: ImpalaMlp [4] -> 2, episode_len 200, BATCH_SIZE 800, 2 trajectories per train"""
    alg = _alg("ImpalaMlp", 2, 200, 800, [4])
    _run_alg(alg, iko.impala_mlp_arch(), 2, 200, 2, (4,), 800)
    s = np.random.default_rng(0).standard_normal(4).astype(np.float32)
    p, v = alg.predict(s)
    assert p.shape == (1, 2) and v.shape == (1, 1) and abs(float(p.sum()) - 1.0) < 1e-5


def test_impala_cnn_two_slices_matches_oracle(xb):
    """uint8 ImpalaCnn, 4 x 50 steps, BATCH_SIZE 150: slices of 150 (128 + 22) and 50 rows"""
    alg = _alg("ImpalaCnn", 4, 50, 150, [84, 84, 4])
    _run_alg(alg, iko.impala_cnn_arch(), 4, 50, 4, (84, 84, 4), 150, clipnorm=40.0, decay=5.12e-9)


def test_graph_replay_equals_eager(xb):
    lib = xb["lib"]
    res = []
    for graph in (True, False):
        alg = _alg("ImpalaCnn", 4, 20, 32, [84, 84, 4], use_cuda_graph=graph)
        out = []
        for c in range(2):
            for tr in _trajs(2, 20, 4, (84, 84, 4), seed=50 + c):
                alg.prepare_data(tr)
            r0 = lib.xtb_graph_replay_count()
            np.random.seed(c)
            loss = alg.train()
            assert lib.xtb_graph_replay_count() - r0 == (1 if graph else 0)
            out.append((loss, alg.pg_adv.cpu().numpy().copy(), alg.target_value.cpu().numpy().copy()))
        res.append((out, np.concatenate([v.ravel() for v in alg.get_weights().values()])))
    (g, gw), (e, ew) = res
    # the first call's V-trace reads the same initial weights through deterministic forwards: bitwise equal
    np.testing.assert_array_equal(g[0][1], e[0][1])
    np.testing.assert_array_equal(g[0][2], e[0][2])
    for (lg, pg, _), (le, pe, _) in zip(g, e):
        assert abs(lg - le) < 1e-4 * max(1.0, abs(le))
        assert rel_err(pg, pe) < 1e-4
    assert l2_rel(gw, ew) < 1e-3


# ------------------------------------------------------------------------------------------- validation
def test_invalid_arguments_launch_nothing(xb):
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = xb["lib"]
    m = _mlp(4)
    net = m.net
    lt, vt = net.tid[m.logit_name], net.tid[m.value_name]
    n = 16
    obs, order = dev(np.zeros((n, 4), np.float32)), dev(np.arange(n, dtype=np.int32))
    y, adv, tv = dev(np.zeros((n, 4), np.float32)), dev(np.zeros(n, np.float32)), dev(np.zeros(n, np.float32))
    loss = torch.zeros(1, device="cuda")

    def fit(**kw):
        a = dict(n=n, fb=8, lt=lt, vt=vt, obs=obs)
        a.update(kw)
        return lib.xtb_impala_keras_fit(net.handle, m.opt.handle, _ptr(a["obs"]), _ptr(order), _ptr(y), _ptr(adv), _ptr(tv),
                                        a["n"], a["fb"], a["lt"], a["vt"], 0.01, _ptr(loss), 0, stream_ptr())
    torch.cuda.synchronize()
    before = lib.xtb_launch_count()
    assert fit(n=0) == -1
    assert fit(fb=0) == -1
    assert fit(fb=net.max_batch + 1, n=net.max_batch + 1) == -1
    assert fit(lt=vt) == -1
    assert fit(vt=lt) == -1                                 # the value head must be 1 wide
    assert fit(lt=99) == -1
    assert fit(obs=None) == -1
    tr = capi.ImpalaTraj(_ptr(obs), _ptr(y), _ptr(y), _ptr(adv), None)
    scratch = dev(np.zeros(n, np.int32))
    assert lib.xtb_impala_keras_train(net.handle, m.opt.handle, tr, 1, n - 1, 8, 8, _ptr(order), _ptr(scratch), 0.99, 0.01,
                                      lt, vt, _ptr(adv), _ptr(tv), _ptr(loss), 0, stream_ptr()) == -1      # done is NULL
    tr.done = _ptr(dev(np.zeros(n, np.uint8)))
    assert lib.xtb_impala_keras_train(net.handle, m.opt.handle, tr, 64, 63, 8, 8, _ptr(order), _ptr(scratch), 0.99, 0.01,
                                      lt, vt, _ptr(adv), _ptr(tv), _ptr(loss), 0, stream_ptr()) == -1      # > max_batch states
    big = _mlp(33)                                          # more actions than the kernels take
    assert lib.xtb_impala_keras_fit(big.net.handle, big.opt.handle, _ptr(obs), _ptr(order), _ptr(y), _ptr(adv), _ptr(tv), n, 8,
                                    big.net.tid[big.logit_name], big.net.tid[big.value_name], 0.01, _ptr(loss), 0,
                                    stream_ptr()) == -1
    hook = capi.GRAD_HOOK(lambda *a: 0)
    capi.check(lib.xtb_set_grad_hook(hook, None))
    try:
        assert fit() == -3 and b"data-parallel" in lib.xtb_last_error()
    finally:
        capi.check(lib.xtb_set_grad_hook(C.cast(None, capi.GRAD_HOOK), None))
    assert lib.xtb_launch_count() == before
    assert fit() == 0


# ------------------------------------------------------------------------------------------- weights
def test_save_load_round_trip(xb, tmp_path):
    m = _cnn(18)
    w = m.get_weights()
    assert list(w) == ["conv2d/kernel", "conv2d/bias", "conv2d_1/kernel", "conv2d_1/bias", "conv2d_2/kernel", "conv2d_2/bias",
                       "dense/kernel", "dense/bias", "output_actions/kernel", "output_actions/bias", "output_value/kernel",
                       "output_value/bias"]
    assert not w["output_value/bias"].any() and w["output_value/kernel"].any()
    x = np.random.default_rng(0).integers(0, 256, (5, 84, 84, 4), dtype=np.uint8)
    path = m.save_model(str(tmp_path / "actor_00001"))
    fresh = _cnn(18, seed=3)
    assert not np.array_equal(fresh.predict([x, None])[0], m.predict([x, None])[0])
    fresh.load_model(path)
    for a, b in zip(fresh.predict([x, None]), m.predict([x, None])):
        np.testing.assert_array_equal(a, b)
    with orc.precision("f64"):
        p, v = iko.ImpalaKerasLearner(iko.impala_cnn_arch(action_dim=18), w).predict(x)
    got = m.predict([x, None])
    assert rel_err(got[0], p) < 1e-3 and rel_err(got[1], v) < 1e-3
