"""The hidden activations past relu / tanh (sigmoid, softsign, softplus, leaky_relu, elu, selu, swish, gelu) on the
device, on the tensor-core and fp32 kernel paths, against float64:

- the layer engine on a subset of test_gpu_layer_sweep.CASES: an s2d first layer, tensor-core convs (SAME, and a tensor
  read by two layers: the `accumulate` epilogue), a dense pair, the split-K dense-4096 forward and an fp32 fallback;
  forward and every weight / bias gradient, under the sweep's bounds.  leaky_relu and selu get the sweep's ReLU
  treatment at their kink: the float64 backward takes the branch of the GPU forward after asserting that it differs from
  the float64 sign only where |pre| < MASK_TIE max|pre|.
- PPO through the plugin API (PpoMlp Categorical and DiagGaussian, PpoCnn 84x84x4): one SGD step against the oracle
  learner with fused heads on and off, predict against the oracle with supplied noise;
- a swish PpoCnn train call on the tensor cores with fused heads is bitwise reproducible;
- xtb_net_create rejects an activation outside the enum without a launch."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import activations_oracle as ao
import gauss_oracle as gor
from oracle import xt_oracle as orc
from test_gpu_kernels import (F32_FLOOR, REL, RELU_FLIP_F32, RELU_FLIP_TC, TC_FWD_BOUND, TC_GRAD_BOUND, _keepalive, dev,  # noqa: F401
                              l2_rel, rel_err, tc_mode, xb)
from test_gpu_layer_sweep import CASES, MASK_TIE, _assert_plan, _gpu_run, _inputs, _plan, _weights
from test_gpu_plugins import alg_cfg
from test_gpu_ppo_gauss import _desc

pytestmark = pytest.mark.gpu

ao.install()


@pytest.fixture(autouse=True)
def _restore_module_config():
    """model / algorithm configs overwrite their modules' globals (import_config, as in the reference): put them back so
    the settings of these tests do not reach the tests that run after them"""
    import sys
    import xingtian_b200  # noqa: F401  (the model and algorithm modules)
    mods = [m for n, m in list(sys.modules.items()) if n.startswith("xingtian_b200") and m is not None]
    saved = [(m, k, v) for m in mods for k, v in vars(m).items() if k.isupper() and isinstance(v, (bool, int, float, str))]
    yield
    for m, k, v in saved:
        setattr(m, k, v)


SUBSET = ["s2d_84x84_k8_valid", "width_10x10_16to48_k3s1_same", "dag_two_tc_convs", "dense_80x48", "dense_4096x16", "fb_cin8"]
KINKED = {"leaky_relu": lambda p: ao.LEAKY_ALPHA * p,
          "selu": lambda p: ao.SELU_SCALE * ao.SELU_ALPHA * torch.expm1(torch.clamp(p, max=0))}


def _act_t(act, p, mask):
    if act in KINKED and mask is not None:
        m = torch.from_numpy(mask).reshape(p.shape)
        pos = p * (ao.SELU_SCALE if act == "selu" else 1.0)
        return torch.where(m, pos, KINKED[act](p))
    return ao.TORCH[act](p)


def _reference(arch, w, obs, dt, act, gh, masks=None):
    """torch-CPU forward in dtype dt with the activation under test: every tensor and the parameter gradients of
    sum_h pre_h . G_h.  A kinked layer takes the branch of masks[name] when given."""
    params = {k: torch.from_numpy(v).to(dt).requires_grad_(True) for k, v in w.items()}
    B = obs.shape[0]
    x = torch.from_numpy(obs).to(dt)
    t, pre = {"obs": x / 255.0 if arch["input_dtype"] == "uint8" else x}, {}
    for name, kind, src, sp in arch["layers"]:
        a = t[src]
        if kind == "conv":
            xin = a.permute(0, 3, 1, 2)
            if sp["pad"] == "same":
                _, pt, pb = orc._same_pad(a.shape[1], sp["k"], sp["s"])
                _, pl, pr = orc._same_pad(a.shape[2], sp["k"], sp["s"])
                xin = F.pad(xin, (pl, pr, pt, pb))
            p = F.conv2d(xin, params[name + "/kernel"].permute(3, 2, 0, 1), params[name + "/bias"], stride=sp["s"]).permute(0, 2, 3, 1)
        else:
            p = a.reshape(B, -1) @ params[name + "/kernel"] + params[name + "/bias"]
        pre[name] = p
        t[name] = _act_t(act, p, None if masks is None else masks.get(name))
    loss = sum((pre[h].reshape(B, -1) * torch.from_numpy(gh[h]).to(dt)).sum() for h in arch["outputs"])
    loss.backward()
    return ({n: v.detach().reshape(B, -1).numpy() for n, v in t.items() if n != "obs"},
            {n: v.detach().reshape(B, -1).numpy() for n, v in pre.items()},
            {k: params[k].grad.numpy() for k in w})


@pytest.mark.parametrize("act", ao.NEW)
@pytest.mark.parametrize("case", SUBSET)
def test_layer_engine(xb, tc_mode, case, act):
    from xingtian_b200.engine import Net
    make, B, max_batch, gather, expect = CASES[case]
    arch = make(act)
    net = Net(arch, max_batch=max_batch)
    _assert_plan(_plan(net, arch), expect)
    w = _weights(arch)
    net.set_weights(w)
    obs, idx, gh = _inputs(arch, B, gather)
    gpu_t, gpu_g = _gpu_run(net, arch, obs, idx, B, gh)
    x = obs[idx] if idx is not None else obs
    masks = None
    if act in KINKED:
        f64_t, pre64, _ = _reference(arch, w, x, torch.float64, act, gh)
        masks = {}
        for n in pre64:
            m = gpu_t[n] > 0
            flip = m != (pre64[n] > 0)
            worst = float(np.abs(pre64[n][flip]).max()) if flip.any() else 0.0
            assert worst < MASK_TIE * float(np.abs(pre64[n]).max()), (n, int(flip.sum()), worst)
            masks[n] = m
    f64_t, _, f64_g = _reference(arch, w, x, torch.float64, act, gh, masks)
    fwd = {n: rel_err(gpu_t[n], f64_t[n]) for n in gpu_t}
    grd = {k: (l2_rel(gpu_g[k], f64_g[k]), rel_err(gpu_g[k], f64_g[k])) for k in w}
    if tc_mode:
        bad = {n: e for n, e in fwd.items() if not e < TC_FWD_BOUND}
        bad.update({k: e for k, e in grd.items() if not (e[0] < TC_GRAD_BOUND and e[1] < REL)})
    else:
        f32_t, _, f32_g = _reference(arch, w, x, torch.float32, act, gh, masks)
        cpu_f = {n: rel_err(f32_t[n], f64_t[n]) for n in fwd}
        cpu_g = {k: l2_rel(f32_g[k], f64_g[k]) for k in w}
        # the fp32 GEMM adds K terms in order; an activation that passes negative pre-activations on (elu at K = 4096:
        # 3.4e-6 against torch-CPU's 5.6e-7) carries more of that into the next layer than relu / tanh do
        bad = {n: (e, cpu_f[n]) for n, e in fwd.items() if not e <= 2 * cpu_f[n] + 2 * F32_FLOOR}
        bad.update({k: (e[0], cpu_g[k]) for k, e in grd.items() if not e[0] <= 2 * cpu_g[k] + F32_FLOOR})
    assert not bad, bad


# ---- PPO through the plugin API
SHAPES = {
    "cartpole": dict(model="PpoMlp", state_dim=[4], A=2, hidden=[64, 64], gauss=False, dtype=np.float32),
    "pendulum": dict(model="PpoMlp", state_dim=[3], A=1, hidden=[64, 64], gauss=True, dtype=np.float32),
    "cnn": dict(model="PpoCnn", state_dim=[84, 84, 4], A=4, hidden=[256], gauss=False, dtype=np.uint8),
}


def _model(shape, act, B):
    import xingtian_b200  # noqa: F401
    from xingtian_b200.registry import Registers
    s = SHAPES[shape]
    cfg = {"BATCH_SIZE": B, "NUM_SGD_ITER": 1, "hidden_sizes": s["hidden"], "activation": act, "init_seed": 3,
           "VF_CLIP": 0.5, "ENTROPY_LOSS": 0.01, "LOSS_CLIPPING": 0.2,
           "action_type": "DiagGaussian" if s["gauss"] else "Categorical"}
    if s["model"] == "PpoMlp":
        cfg["VF_SHARE_LAYERS"] = False
    info = {"state_dim": s["state_dim"], "action_dim": s["A"], "model_config": cfg}
    if s["dtype"] == np.uint8:
        info["input_dtype"] = "uint8"
    return Registers.model[s["model"]](info)


def _arch(shape, act):
    s = SHAPES[shape]
    if s["model"] == "PpoCnn":
        a = orc.ppo_cnn_arch(action_dim=s["A"], hidden_sizes=tuple(s["hidden"]), activation=act)
    else:
        a = orc.ppo_mlp_arch(state_dim=tuple(s["state_dim"]), action_dim=s["A"], hidden_sizes=tuple(s["hidden"]), activation=act)
    return gor.with_logstd(a) if s["gauss"] else a


def _step_data(shape, arch, w, B, seed):
    s = SHAPES[shape]
    rng = np.random.default_rng(seed)
    if s["dtype"] == np.uint8:
        obs = rng.integers(0, 256, (B,) + tuple(s["state_dim"]), dtype=np.uint8)
    else:
        obs = rng.standard_normal((B,) + tuple(s["state_dim"])).astype(np.float32)
    if s["gauss"]:
        mean, v = [t.detach().numpy() for t in gor.forward(arch, w, obs)]
        act = (mean + np.exp(w["pi_logstd"]) * 1.2 * rng.standard_normal((B, s["A"]))).astype(np.float32)
        lp = gor.log_prob(torch.from_numpy(act), torch.from_numpy(mean), torch.from_numpy(w["pi_logstd"])).numpy()
    else:
        logits, v = [t.detach().numpy() for t in orc.forward(arch, w, obs)]
        act = rng.integers(0, s["A"], B).astype(np.int32)
        lp = orc.categorical_logp(torch.from_numpy(logits), torch.from_numpy(act)).numpy().reshape(B, 1)
    old_logp = (lp + 0.5 * rng.standard_normal((B, 1))).astype(np.float32)
    label = [act, old_logp, rng.standard_normal((B, 1)).astype(np.float32),
             (v + 1.5 * rng.standard_normal((B, 1))).astype(np.float32), rng.standard_normal((B, 1)).astype(np.float32)]
    return obs, label


def _oracle_step(shape, arch, w, obs, label, B, dt):
    learner = gor.PpoLearner if SHAPES[shape]["gauss"] else orc.PpoLearner
    with orc.precision(dt):
        ref = learner(arch, w, batch_size=B, ent_coef=0.01, clip_ratio=0.2, num_sgd_iter=1, vf_clip=0.5)
        loss, grads = ref.loss_and_grads(obs, *label)
        return float(loss.detach()), {k: g.detach().numpy() for k, g in zip(ref.names, grads)}


@pytest.mark.parametrize("act", ao.NEW)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_ppo_train_step_against_float64(xb, tc_mode, shape, act):
    """one SGD step with fused heads on and off: loss and every gradient at most 4x torch-CPU fp32's distance from
    float64 (+ the floor of test_gpu_ppo_gauss; leaky_relu / selu: the ReLU flip allowance of the PPO tests), and the
    two modes agree to rounding"""
    lib = xb["lib"]
    B = 200 if shape != "cnn" else 64
    got = {}
    try:
        for fuse in (1, 0):
            lib.xtb_set_fuse_heads(fuse)
            m = _model(shape, act, B)
            w = m.get_weights()
            if SHAPES[shape]["gauss"]:
                w["pi_logstd"] = np.full((1, SHAPES[shape]["A"]), -0.3, np.float32)
                m.set_weights(w)
            arch = _arch(shape, act)
            obs, label = _step_data(shape, arch, w, B, seed=7)
            np.random.seed(0)
            m.train([obs], label)
            got[fuse] = (float(m.last_losses[0]), m.net.get_weights(m.net.grads))
    finally:
        lib.xtb_set_fuse_heads(1)
    l64, g64 = _oracle_step(shape, arch, w, obs, label, B, "f64")
    l32, g32 = _oracle_step(shape, arch, w, obs, label, B, "f32")
    floor = (6e-5 if tc_mode == 1 else 1e-5) * max(1.0, np.sqrt(B / 128.0))
    if act in KINKED:       # units at the kink take the other slope under the forward's rounding, as ReLU units do
        floor = max(floor, RELU_FLIP_TC if tc_mode == 1 else RELU_FLIP_F32)
    for fuse, (loss, g) in got.items():
        assert abs(loss - l64) <= 4 * abs(l32 - l64) + floor * max(1.0, abs(l64)), (fuse, loss, l64, l32)
        bad = {k: (l2_rel(g[k], g64[k]), l2_rel(g32[k], g64[k])) for k in g64
               if not l2_rel(g[k], g64[k]) <= 4 * l2_rel(g32[k], g64[k]) + floor}
        assert not bad, (fuse, bad)
    assert abs(got[1][0] - got[0][0]) <= 1e-5 * max(1.0, abs(got[0][0]))
    for k in got[0][1]:
        assert l2_rel(got[1][1][k], got[0][1][k]) < 1e-4, k


@pytest.mark.parametrize("act", ao.NEW)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_predict_against_oracle(xb, tc_mode, shape, act):
    """predict with supplied uniforms / normals: log-probs and values within 1e-3 of the float64 oracle, actions exact
    (Categorical) or within 1e-3 (Gaussian: the action is mean + std * n)"""
    s = SHAPES[shape]
    B = 37
    m = _model(shape, act, B)
    arch = _arch(shape, act)
    w = m.get_weights()
    obs, _ = _step_data(shape, arch, w, B, seed=9)
    rng = np.random.default_rng(3)
    w64 = {k: v.astype(np.float64) for k, v in w.items()}
    if s["gauss"]:
        n = rng.standard_normal((B, s["A"])).astype(np.float32)
        a, lp, v = m.predict(obs, normals=n)
        with orc.precision("f64"):
            ra, rlp, rv = gor.predict(arch, w64, obs.astype(np.float64), n.astype(np.float64))
        assert rel_err(a, ra) < 1e-3
    else:
        u = (rng.random((B, s["A"])) * 0.99 + 0.005).astype(np.float32)
        a, lp, v = m.predict(obs, uniforms=u)
        with orc.precision("f64"):
            ra, rlp, rv = orc.ppo_predict(arch, w64, obs if obs.dtype == np.uint8 else obs.astype(np.float64), u)
        np.testing.assert_array_equal(np.asarray(a), np.asarray(ra))
    assert rel_err(np.ravel(lp), np.ravel(rlp)) < 1e-3 and rel_err(np.ravel(v), np.ravel(rv)) < 1e-3


def test_swish_cnn_training_is_bitwise_reproducible(xb):
    """tensor-core trunk, fused heads: the swish backward reads the retained pre-activation, and the step stays free of
    atomics, so two runs from the same weights and shuffle stream are identical"""
    import xingtian_b200 as xtb
    lib = xb["lib"]
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(1)
    info = {"actor": {"model_name": "PpoCnn", "state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8",
                      "model_config": {"BATCH_SIZE": 320, "ENTROPY_LOSS": 0.003, "LOSS_CLIPPING": 0.1, "LR": 0.00025,
                                       "NUM_SGD_ITER": 2, "hidden_sizes": [256], "activation": "swish", "init_seed": 0}}}
    ro = orc.synth_ppo_rollout(5, 4, 128)
    runs = []
    try:
        for _ in range(2):
            alg = xtb.alg_builder("PPO", info, alg_cfg(instance_num=4))
            for e in range(4):
                sl = slice(e * 128, (e + 1) * 128)
                alg.prepare_data(dict(cur_state=ro["obs"][sl], action=ro["action"][sl], logp=ro["logp"][sl],
                                      value=ro["value"][e], reward=ro["reward"][sl], done=ro["done"][sl]))
            np.random.seed(21)
            alg.train()
            runs.append((np.asarray(alg.actor.last_losses, np.float32), alg.get_weights()))
    finally:
        lib.xtb_set_tc_mode(old)
    assert np.array_equal(runs[0][0], runs[1][0]), (runs[0][0], runs[1][0])
    for k in runs[0][1]:
        assert np.array_equal(runs[0][1][k], runs[1][1][k]), k


def test_create_rejects_unknown_activation(xb):
    capi, lib = xb["capi"], xb["lib"]
    D = capi.DENSE
    for act in (11, -1):
        before = lib.xtb_launch_count()
        h = C.c_void_p()
        assert lib.xtb_net_create(C.byref(_desc(capi, [(D, 0, act, 64), (D, 1, 0, 3)])), 8, C.byref(h)) == -1, act
        assert lib.xtb_launch_count() == before
    h = C.c_void_p()
    assert lib.xtb_net_create(C.byref(_desc(capi, [(D, 0, 10, 64), (D, 1, 0, 3)])), 8, C.byref(h)) == 0
    lib.xtb_net_destroy(h)
