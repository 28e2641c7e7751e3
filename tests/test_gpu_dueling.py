"""The dueling Q head (layer kind "dueling", XTB_DUELING) on the device: the layer engine against float64 on both kernel
paths, descriptor validation, DQN + DqnCnn / DqnMlp with model_config {dueling: True} against the oracle learner, the
fused dueling TD step against the layer-by-layer one, and weight I/O.

Engine parity uses the bounds of test_gpu_layer_sweep (tensor-core path: forward max-rel < TC_FWD_BOUND, gradient
L2-rel < TC_GRAD_BOUND and max-rel < 1e-3; fp32 path: at most 2x torch-CPU fp32's distance from float64 + F32_FLOOR),
with random head gradients injected at the combine tensor and the GPU ReLU mask in the float64 backward."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import dueling_oracle as dor
from oracle import xt_oracle as orc
from parity_record import record as _record
from test_gpu_kernels import (F32_FLOOR, REL, TC_FWD_BOUND, TC_GRAD_BOUND, _keepalive, dev, l2_rel, rel_err,  # noqa: F401
                              tc_mode, xb)
from test_gpu_layer_sweep import MASK_TIE, _stemmed
from test_gpu_plugins import alg_cfg

pytestmark = pytest.mark.gpu


def _dense(name, src, n, act):
    return (name, "dense", src, dict(n=n, act=act))


def _cnn(A, act, extra=False):
    """DqnCnn-shaped: s2d stem -> conv -> dense 256 (tensor cores) -> value A, adv 1 -> combine"""
    layers = [("c", "conv", "x", dict(k=3, s=1, cout=64, pad="valid", act=act)), _dense("h", "c", 256, act),
              _dense("value", "h", A, None), _dense("adv", "h", 1, None), ("q", "dueling", ("value", "adv"), {})]
    outs = ["q"]
    if extra:   # both combine sources also feed another head: the data gradient accumulates into them
        layers += [_dense("x1", "value", 16, act), _dense("x2", "adv", 8, act)]
        outs += ["x1", "x2"]
    return _stemmed((6, 6), 32, act, layers, outs)


def _mlp(A, act):
    """DqnMlp-shaped: float state 4 -> dense 128 -> value A, adv 1 -> combine"""
    return dict(input_dtype="float32", state_dim=(4,), scale=1.0, outputs=["q"], layers=[
        _dense("h", "obs", 128, act), _dense("value", "h", A, None), _dense("adv", "h", 1, None),
        ("q", "dueling", ("value", "adv"), {})])


def _weights(arch, seed=11):
    w = dor.init_weights(arch, seed=seed)
    rng = np.random.default_rng(seed + 1)
    for k in w:                                   # non-zero biases so the bias paths are exercised
        if k.endswith("/bias"):
            w[k] = (rng.standard_normal(w[k].shape) * 0.05).astype(np.float32)
    return w


def _reference(arch, w, x, dt, gh=None, masks=None):
    """every tensor and (gh given) the parameter gradients of sum_h pre_h . G_h in torch-CPU `dt`"""
    params = {k: torch.from_numpy(v).to(dt).requires_grad_(gh is not None) for k, v in w.items()}
    B = x.shape[0]
    xt = torch.from_numpy(x).to(dt)
    t, pre = {"obs": xt / 255.0 if arch["input_dtype"] == "uint8" else xt}, {}
    for name, kind, src, sp in arch["layers"]:
        if kind == "dueling":
            p = dor.combine(t[src[0]], t[src[1]])
        elif kind == "conv":
            a = t[src].permute(0, 3, 1, 2)
            p = torch.nn.functional.conv2d(a, params[name + "/kernel"].permute(3, 2, 0, 1), params[name + "/bias"],
                                           stride=sp["s"]).permute(0, 2, 3, 1)
        else:
            p = t[src].reshape(B, -1) @ params[name + "/kernel"] + params[name + "/bias"]
        pre[name] = p
        act = sp.get("act")
        if act == "relu":
            t[name] = p * torch.from_numpy(masks[name]).to(dt).reshape(p.shape) if masks is not None else torch.relu(p)
        else:
            t[name] = torch.tanh(p) if act == "tanh" else p
    outs = {n: v.detach().reshape(B, -1).numpy() for n, v in t.items() if n != "obs"}
    pres = {n: v.detach().reshape(B, -1).numpy() for n, v in pre.items()}
    if gh is None:
        return outs, pres, None
    loss = sum((pre[h].reshape(B, -1) * torch.from_numpy(gh[h]).to(dt)).sum() for h in arch["outputs"])
    loss.backward()
    return outs, pres, {k: params[k].grad.numpy() for k in w}


def _engine_parity(arch, B, tc, tag):
    from xingtian_b200.engine import Net
    net = Net(arch, max_batch=B)
    w = _weights(arch)
    net.set_weights(w)
    rng = np.random.default_rng(B + 7)
    shape = (B,) + tuple(arch["state_dim"])
    obs = rng.integers(0, 256, shape, dtype=np.uint8) if arch["input_dtype"] == "uint8" else rng.standard_normal(shape).astype(np.float32)
    sizes = dor.tensor_shapes(arch)
    gh = {h: rng.standard_normal((B, int(np.prod(sizes[h])))).astype(np.float32) for h in arch["outputs"]}
    obs_d = dev(obs)
    net.forward(obs_d, B)
    gpu_t = {n: net.tensor(n)[:B].cpu().numpy() for n, _, _, _ in arch["layers"]}
    for h in arch["outputs"]:
        net.tensor_grad(h)[:B].copy_(dev(gh[h]))
    net.backward(obs_d, B, arch["outputs"])
    gpu_g = net.get_weights(net.grads)
    assert list(gpu_g) == list(w)
    # float64 reference, ReLU through the GPU mask where the sign is a tie
    f64_t, pre64, _ = _reference(arch, w, obs, torch.float64)
    masks = {}
    for n, _, _, sp in arch["layers"]:
        if sp.get("act") == "relu":
            m = gpu_t[n] > 0
            flip = m != (pre64[n] > 0)
            worst = float(np.abs(pre64[n][flip]).max()) if flip.any() else 0.0
            assert worst < MASK_TIE * float(np.abs(pre64[n]).max()), (n, int(flip.sum()), worst)
            masks[n] = m
    _, _, f64_g = _reference(arch, w, obs, torch.float64, gh, masks)
    fwd = {n: rel_err(gpu_t[n], f64_t[n]) for n in gpu_t}
    grd = {k: (l2_rel(gpu_g[k], f64_g[k]), rel_err(gpu_g[k], f64_g[k])) for k in w}
    plan_tc = any(net.layer_plan(i)["tc"] for i in range(len(arch["layers"])))
    if tc and plan_tc:
        bad = {n: e for n, e in fwd.items() if not e < TC_FWD_BOUND}
        bad.update({k: e for k, e in grd.items() if not (e[0] < TC_GRAD_BOUND and e[1] < REL)})
    else:
        f32_t, _, f32_g = _reference(arch, w, obs, torch.float32, gh, masks)
        cpu_f = {n: rel_err(f32_t[n], f64_t[n]) for n in fwd}
        cpu_g = {k: l2_rel(f32_g[k], f64_g[k]) for k in w}
        # The fp32 weight-gradient GEMM adds the batch sequentially within each K slice, torch-CPU pairwise.  A bias
        # gradient whose per-sample terms have random sign (the value stream at A = 2: (g0 - g1) / 2) is ~sqrt(B) smaller
        # than the sum of its magnitudes, so its relative error grows like sqrt(B): observed 2.4-2.7e-6 at B = 512.
        floor = F32_FLOOR * max(1.0, np.sqrt(B / 128.0))
        bad = {n: (e, cpu_f[n]) for n, e in fwd.items() if not e <= 2 * cpu_f[n] + F32_FLOOR}
        bad.update({k: (e[0], cpu_g[k]) for k, e in grd.items() if not e[0] <= 2 * cpu_g[k] + floor})
    _record(tag, {"forward_max_rel": {n: "%.2e" % e for n, e in fwd.items()},
                  "grad_l2_rel,max_rel": {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in grd.items()}})
    assert not bad, bad
    return net


@pytest.mark.parametrize("B", [1, 37, 512])
@pytest.mark.parametrize("A", [2, 4, 18])
@pytest.mark.parametrize("act", ["tanh", "relu"])
@pytest.mark.parametrize("shape", ["cnn", "mlp"])
def test_dueling_engine_parity(xb, tc_mode, shape, act, A, B):
    arch = _cnn(A, act) if shape == "cnn" else _mlp(A, act)
    net = _engine_parity(arch, B, tc_mode, "dueling/%s/%s/A%d/B%d/%s" % (shape, act, A, B, "tc" if tc_mode else "fp32"))
    plan = net.layer_plan(len(arch["layers"]) - 1)
    assert plan["kind"] == "dueling" and not plan["tc"]
    if shape == "cnn":
        assert net.layer_plan(2)["tc"]          # the hidden dense layer runs on the tensor cores


@pytest.mark.parametrize("act", ["tanh", "relu"])
def test_dueling_sources_with_a_second_consumer(xb, tc_mode, act):
    """value and adv also feed another layer: the combine's data gradient adds to what that layer wrote"""
    _engine_parity(_cnn(4, act, extra=True), 37, tc_mode, "dueling/extra/%s/%s" % (act, "tc" if tc_mode else "fp32"))


def _desc(layers):
    from xingtian_b200 import capi
    d = capi.NetDesc()
    d.input_u8, d.scale, d.in_h, d.in_w, d.in_c = 0, 1.0, 1, 1, 8
    d.n_layers = len(layers)
    for i, (kind, src, k, cout) in enumerate(layers):
        d.layers[i].kind, d.layers[i].src, d.layers[i].k, d.layers[i].cout = kind, src, k, cout
    return d


@pytest.mark.parametrize("bad", ["obs_value", "obs_adv", "later_adv", "adv_not_1_wide"])
def test_dueling_bad_descriptors(xb, bad):
    from xingtian_b200 import capi
    lib = xb["lib"]
    D, DU = capi.DENSE, capi.DUELING
    base = [(D, 0, 0, 16), (D, 1, 0, 4), (D, 1, 0, 1)]          # tensors 1: hidden, 2: value (4), 3: adv (1)
    duel = {"obs_value": (DU, 0, 3, 0), "obs_adv": (DU, 2, 0, 0), "later_adv": (DU, 2, 5, 0), "adv_not_1_wide": (DU, 2, 1, 0)}[bad]
    layers = base + [duel] + [(D, 2, 0, 1)]
    h = C.c_void_p()
    torch.cuda.synchronize()
    before = lib.xtb_launch_count()
    rc = lib.xtb_net_create(C.byref(_desc(layers)), 8, C.byref(h))
    assert rc == -1 and not h.value, rc            # XTB_ERR_ARG
    assert b"dueling" in lib.xtb_last_error()
    assert lib.xtb_launch_count() == before
    ok = C.c_void_p()
    assert lib.xtb_net_create(C.byref(_desc(base + [(DU, 2, 3, 0)])), 8, C.byref(ok)) == 0
    assert lib.xtb_net_tensor_size(ok, 4) == 4
    kr, nc = C.c_int(-1), C.c_int(-1)
    assert lib.xtb_net_layer_params(ok, 3, None, None, C.byref(kr), C.byref(nc)) == 0 and (kr.value, nc.value) == (0, 0)
    assert lib.xtb_net_param_count(ok) == (8 * 16 + 16) + (16 * 4 + 4) + (16 + 1)
    lib.xtb_net_destroy(ok)


# ------------------------------------------------------------------------------------------- DQN plugin
@pytest.fixture(autouse=True)
def _restore_dqn_config():
    """import_config writes the algorithm / model config into module globals (as the reference does): put them back so
    N_STEP, HUBER_DELTA, BUFFER_SIZE, ... set here do not leak into later tests"""
    from xingtian_b200.algorithm import dqn as alg_mod
    from xingtian_b200.model import dqn as model_mod
    saved = [(m, {k: v for k, v in vars(m).items() if k.isupper()}) for m in (alg_mod, model_mod)]
    yield
    for m, d in saved:
        for k in [k for k in vars(m) if k.isupper() and k not in d]:
            delattr(m, k)
        for k, v in d.items():
            setattr(m, k, v)


def _dqn_alg(A=4, batch=32, seed=5, **kw):
    import xingtian_b200 as xb_
    info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": A,
                      "model_config": {"LR": 0.00015, "init_seed": seed, "dueling": True}}}
    n = max(48, batch + 16)
    cfg = dict(instance_num=2, prepare_times_per_train=4, learning_starts=n - 8, BUFFER_SIZE=n + 16, BATCH_SIZE=batch,
               TARGET_UPDATE_FREQ=2)
    cfg.update(kw)
    return xb_.alg_builder("DQN", info, alg_cfg(**cfg)), n


def _transitions(n, A, seed=0):
    rng = np.random.default_rng(seed)
    s = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8); s2 = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)
    a = rng.integers(0, A, n); r = np.sign(rng.standard_normal(n)); d = rng.random(n) < 0.1
    return s, a, r, s2, d


def _fill(alg, s, a, r, s2, d):
    for i in range(len(s)):
        alg.prepare_data(dict(cur_state=[s[i]], action=[a[i]], reward=[r[i]], next_state=[s2[i]], done=[d[i]]))


def _run_vs_oracle(alg, n, batch, steps, A, double=False, tol=5e-3, upd_tol=5e-2):
    s, a, r, s2, d = _transitions(n, A)
    w0 = alg.get_weights()
    arch = dor.dqn_cnn_arch(action_dim=A, dueling=True)
    assert list(w0) == list(dor.param_shapes(arch))
    ref = dor.DqnLearner(arch, w0, lr=0.00015, clipnorm=10.0, target_update_freq=2, double_dqn=double)
    _fill(alg, s, a, r, s2, d)
    for step in range(steps):
        random.seed(step)
        loss = alg.train()
        random.seed(step)
        picks = random.sample(range(n), batch)
        ref_loss = ref.train(s[picks], a[picks], r[picks], s2[picks], d[picks])
        assert abs(loss - ref_loss) < tol * max(1.0, abs(ref_loss)), (step, loss, ref_loss)
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0]); rupd = np.concatenate([(r1[k] - w0[k]).ravel() for k in w0])
    assert l2_rel(upd, rupd) < upd_tol
    return s, ref


def test_dueling_dqn_train_matches_oracle(xb):
    """3 steps at B = 32, then Algorithm.predict and the keras-style actor.train(state, y)"""
    alg, n = _dqn_alg()
    assert sum(v.size for v in alg.get_weights().values()) == 882341
    s, ref = _run_vs_oracle(alg, n, 32, 3, 4)
    assert alg.predict(s[0]) == int(np.argmax(ref.predict(s[:1])[0]))
    y = ref.predict(s[:8]); y[:, 1] += 1.0
    assert abs(alg.actor.train(s[:8], y) - 0.25) < 0.05


def test_dueling_dqn_c4_size_matches_oracle(xb):
    alg, n = _dqn_alg(batch=512)
    _run_vs_oracle(alg, n, 512, 2, 4)


def test_dueling_double_dqn_matches_oracle(xb):
    alg, n = _dqn_alg(double_dqn=True)
    _run_vs_oracle(alg, n, 32, 1, 4, double=True)


def test_dueling_nstep_huber_step_matches_oracle(xb):
    """one N_STEP = 3, HUBER_DELTA = 1 step (n-step bootstrap discounts per row, Huber loss) through the plugin's online
    and target models, against the oracle learner"""
    alg, _ = _dqn_alg(N_STEP=3, HUBER_DELTA=1.0)
    assert alg.n_step == 3 and alg.huber_delta == 1.0
    model, n = alg.actor, 32
    A = model.action_dim
    s, a, r, s2, d = _transitions(n, A, seed=3)
    rng = np.random.default_rng(4)
    disc = np.where(d, 0.0, 0.99 ** 3).astype(np.float32)
    r = (r + rng.standard_normal(n)).astype(np.float32)
    w0 = model.get_weights()
    arch = dor.dqn_cnn_arch(action_dim=A, dueling=True)
    ref = dor.DqnLearner(arch, w0, lr=0.00015, clipnorm=10.0, target_update_freq=1000)
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    model.train_td_device(alg.target_actor, dev(s), dev(a.astype(np.int32)), dev(r), dev(s2), dev(d.astype(np.uint8)), n, 0.99,
                          loss, disc=dev(disc), huber_delta=alg.huber_delta)
    got = float(loss.cpu()[0])
    want = ref.train(s, a, r, s2, d, disc=disc, huber=1.0)
    assert abs(got - want) < 5e-3 * max(1.0, abs(want)), (got, want)
    w1, r1 = model.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0]); rupd = np.concatenate([(r1[k] - w0[k]).ravel() for k in w0])
    assert l2_rel(upd, rupd) < 5e-2


# ------------------------------------------------------------------------------------------- fused vs layer by layer
def _one_td_step(A, fuse, n=512, eager=False):
    from xingtian_b200 import capi
    from xingtian_b200.model.dqn import DqnCnn
    lib = capi.lib()
    mk = lambda: DqnCnn({"state_dim": [84, 84, 4], "action_dim": A,   # noqa: E731
                         "model_config": {"dueling": True, "init_seed": 9, "LR": 0.00015, "use_cuda_graph": not eager}})
    model, tgt = mk(), mk()
    w0 = model.get_weights()
    ring = 2 * n
    s, a, r, s2, d = _transitions(ring, A, seed=11)
    idx = dev(np.random.default_rng(12).permutation(ring)[:n].astype(np.int32))
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    lib.xtb_set_fuse_heads(1 if fuse else 0)
    try:
        torch.cuda.synchronize()
        before = lib.xtb_launch_count()
        model.train_td_device(tgt, dev(s), dev(a.astype(np.int32)), dev(r.astype(np.float32)), dev(s2), dev(d.astype(np.uint8)),
                              n, 0.99, loss, idx=idx)
        torch.cuda.synchronize()
        launches = lib.xtb_launch_count() - before
    finally:
        lib.xtb_set_fuse_heads(1)
    picks = idx.cpu().numpy()
    return float(loss.cpu()[0]), w0, model.get_weights(), launches, (s[picks], a[picks], r[picks], s2[picks], d[picks])


@pytest.mark.parametrize("A", [4, 6, 9])
def test_fused_dueling_step_matches_layer_by_layer(xb, A):
    lf, w0, wf, nf, batch = _one_td_step(A, True, eager=True)
    lu, w0u, wu, nu, _ = _one_td_step(A, False, eager=True)
    assert all(np.array_equal(w0[k], w0u[k]) for k in w0)
    if A <= 8:
        assert nf < nu, (nf, nu)      # the fused kernel ran
    else:
        assert nf == nu, (nf, nu)     # beyond the heads-kernel limits: the layer-by-layer step
    assert abs(lf - lu) < 1e-4 * max(1.0, abs(lu)), (lf, lu)
    upf = np.concatenate([(wf[k] - w0[k]).ravel() for k in w0]); upu = np.concatenate([(wu[k] - w0[k]).ravel() for k in w0])
    assert l2_rel(upf, upu) < 1e-2
    arch = dor.dqn_cnn_arch(action_dim=A, dueling=True)
    ref = dor.DqnLearner(arch, w0, lr=0.00015, clipnorm=10.0, target_update_freq=1000)
    with orc.precision("f64"):
        ref = dor.DqnLearner(arch, w0, lr=0.00015, clipnorm=10.0, target_update_freq=1000)
        rl = ref.train(*batch)
        rw = ref.weights()
    rup = np.concatenate([(rw[k] - w0[k]).ravel() for k in w0])
    for loss, up in ((lf, upf), (lu, upu)):
        assert abs(loss - rl) < 5e-3 * max(1.0, abs(rl)), (loss, rl)
        assert l2_rel(up, rup) < 5e-2
    _record("dueling/fused_vs_layers/A%d" % A, {"launches": [nf, nu], "loss": [lf, lu, rl],
                                                "upd_l2_rel(fused,layers)": ["%.2e" % l2_rel(upf, rup), "%.2e" % l2_rel(upu, rup)]})


# ------------------------------------------------------------------------------------------- weights
def test_dueling_weight_io(xb, tmp_path):
    from xingtian_b200.model.dqn import DqnCnn, DqnMlp
    m = DqnCnn({"state_dim": [84, 84, 4], "action_dim": 18, "model_config": {"dueling": True, "init_seed": 2}})
    w = m.get_weights()
    assert list(w) == ["conv2d/kernel", "conv2d/bias", "conv2d_1/kernel", "conv2d_1/bias", "conv2d_2/kernel", "conv2d_2/bias",
                       "dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias", "dense_2/kernel", "dense_2/bias"]
    assert w["dense_2/kernel"].shape == (256, 1) and not w["dense_2/bias"].any() and w["dense_2/kernel"].any()
    x = np.random.default_rng(0).integers(0, 256, (5, 84, 84, 4), dtype=np.uint8)
    path = m.save_model(str(tmp_path / "actor_00001"))
    fresh = DqnCnn({"state_dim": [84, 84, 4], "action_dim": 18, "model_config": {"dueling": True, "init_seed": 3}})
    assert not np.array_equal(fresh.predict(x), m.predict(x))
    fresh.load_model(path)
    np.testing.assert_array_equal(fresh.predict(x), m.predict(x))
    q = dor.forward(dor.dqn_cnn_arch(action_dim=18, dueling=True), w, x)[0].numpy()
    assert rel_err(m.predict(x), q) < 1e-3
    mlp = DqnMlp({"state_dim": [4], "action_dim": 2, "model_config": {"dueling": True, "init_seed": 1}})
    ref = dor.init_weights(dor.dqn_mlp_arch(dueling=True), seed=4)
    mlp.set_weights(dict(ref))
    got = mlp.get_weights()
    assert list(got) == ["dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias", "dense_2/kernel", "dense_2/bias"]
    assert all(np.array_equal(got[k], ref[k]) for k in ref)
    xs = np.random.default_rng(1).standard_normal((7, 4)).astype(np.float32)
    assert rel_err(mlp.predict(xs), dor.forward(dor.dqn_mlp_arch(dueling=True), ref, xs)[0].numpy()) < 1e-5
