"""Parity of every CUDA kernel (through the C-ABI) with the CPU oracle on seeded inputs.

Tolerances: bit-exact for action indices on shared noise; fp results within 1e-3 relative
(BASELINE.json north_star), measured as max|gpu-ref| / max(max|ref|, floor)."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import xt_oracle as orc  # noqa: E402

REL = 1e-3


def rel_err(a, b, floor=1e-6):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), floor))


@pytest.fixture(scope="module")
def xb():
    import xingtian_b200 as pkg
    from xingtian_b200 import capi, engine
    assert torch.cuda.is_available()
    return dict(pkg=pkg, capi=capi, engine=engine, lib=capi.lib())


_KEEP = []   # device tensors must outlive the raw pointers handed to the C-ABI


@pytest.fixture(autouse=True)
def _keepalive():
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    t = t.cuda()
    _KEEP.append(t)
    return t


@contextlib.contextmanager
def one_rank_comm():
    """A one-rank NCCL communicator installed for the duration: the library runs its data-parallel paths on one GPU"""
    from xingtian_b200 import capi, engine
    lib = capi.lib()
    path = engine._nccl_path()
    path = path.encode() if path else None
    ident = (C.c_ubyte * 128)()
    capi.check(lib.xtb_comm_unique_id(path, ident))
    h = C.c_void_p()
    capi.check(lib.xtb_comm_create(path, ident, 0, 1, C.byref(h)))
    capi.check(lib.xtb_set_grad_comm(h))
    try:
        yield
    finally:
        capi.check(lib.xtb_set_grad_comm(None))
        lib.xtb_comm_destroy(h)


# ------------------------------------------------------------------------------------------- GAE
@pytest.mark.parametrize("E,T", [(1, 128), (32, 128), (512, 128), (3, 200), (5, 7), (2, 1), (4, 33)])
def test_gae_matches_oracle(xb, E, T):
    from xingtian_b200.engine import _ptr, stream_ptr
    ro = orc.synth_ppo_rollout(1, E, T, state_dim=(1,), dtype=np.float32)
    rew = ro["reward"].reshape(E, T)
    done = ro["done"].reshape(E, T)
    val = ro["value"]
    adv_ref = np.zeros((E, T)); tv_ref = np.zeros((E, T))
    for e in range(E):
        a, ov, tv = orc.gae(val[e], rew[e], done[e])
        adv_ref[e], tv_ref[e] = a[:, 0], tv[:, 0]
    v_d, r_d, d_d = dev(val.reshape(E, T + 1)), dev(rew.astype(np.float32)), dev(done.view(np.uint8))
    adv = torch.empty(E, T, device="cuda"); ov = torch.empty(E, T, device="cuda"); tv = torch.empty(E, T, device="cuda")
    xb["capi"].check(xb["lib"].xtb_gae(_ptr(v_d), _ptr(r_d), _ptr(d_d), E, T, 0.99, 0.95, 0, _ptr(adv), _ptr(ov), _ptr(tv), stream_ptr()))
    assert rel_err(adv.cpu().numpy(), adv_ref) < REL
    assert rel_err(tv.cpu().numpy(), tv_ref) < REL
    np.testing.assert_array_equal(ov.cpu().numpy(), val[:, :T, 0])


def test_gae_sign_clip_and_empty(xb):
    from xingtian_b200.engine import _ptr, stream_ptr
    E, T = 4, 64
    rng = np.random.default_rng(3)
    rew = rng.normal(0, 3, (E, T))
    done = rng.random((E, T)) < 0.05
    val = rng.standard_normal((E, T + 1, 1)).astype(np.float32)
    ref = np.stack([orc.gae(val[e], np.sign(rew[e]), done[e])[0][:, 0] for e in range(E)])
    adv = torch.empty(E, T, device="cuda"); ov = torch.empty_like(adv); tv = torch.empty_like(adv)
    xb["capi"].check(xb["lib"].xtb_gae(_ptr(dev(val.reshape(E, T + 1))), _ptr(dev(rew.astype(np.float32))), _ptr(dev(done.view(np.uint8))),
                                      E, T, 0.99, 0.95, 1, _ptr(adv), _ptr(ov), _ptr(tv), stream_ptr()))
    assert rel_err(adv.cpu().numpy(), ref) < REL
    # empty rollout is a no-op, not an error
    assert xb["lib"].xtb_gae(_ptr(adv), _ptr(adv), _ptr(dev(done.view(np.uint8))), 0, 0, 0.99, 0.95, 0, _ptr(adv), _ptr(ov), _ptr(tv), stream_ptr()) == 0
    # null pointer is an error with a message
    assert xb["lib"].xtb_gae(None, None, None, 1, 1, 0.99, 0.95, 0, None, None, None, None) < 0
    assert b"null" in xb["lib"].xtb_last_error()


# ------------------------------------------------------------------------------------------- sampling
@pytest.mark.parametrize("B,A", [(1, 4), (32, 4), (513, 6), (64, 18)])
def test_sampling_bit_exact_on_shared_noise(xb, B, A):
    from xingtian_b200.engine import _ptr, stream_ptr
    rng = np.random.default_rng(B * 31 + A)
    logits = rng.standard_normal((B, A)).astype(np.float32) * 2
    u = rng.random((B, A)).astype(np.float32) * 0.999 + 0.0005
    act = torch.empty(B, dtype=torch.int32, device="cuda"); lp = torch.empty(B, device="cuda")
    xb["capi"].check(xb["lib"].xtb_categorical_sample(_ptr(dev(logits)), B, A, _ptr(dev(u)), 0, 0, _ptr(act), _ptr(lp), stream_ptr()))
    ref = orc.gumbel_argmax(logits, u)
    got = act.cpu().numpy()
    # expf/logf on the device differ from numpy by ulps: a mismatch is only legal on a near-tie
    g = -np.log(-np.log(u))
    s = np.sort(logits + g, axis=1)
    gap = s[:, -1] - s[:, -2]
    bad = (got != ref) & (gap > 1e-4)
    assert not bad.any()
    assert (got == ref).mean() > 0.99
    ref_lp = orc.categorical_logp(torch.from_numpy(logits), torch.from_numpy(got)).numpy()[:, 0]
    assert rel_err(lp.cpu().numpy(), ref_lp) < REL
    # internal Philox stream == oracle's Philox restatement (bit exact uniforms -> same actions)
    act2 = torch.empty(B, dtype=torch.int32, device="cuda")
    xb["capi"].check(xb["lib"].xtb_categorical_sample(_ptr(dev(logits)), B, A, None, C.c_uint64(1234567), C.c_uint64(42), _ptr(act2), _ptr(lp), stream_ptr()))
    u2 = orc.philox_uniforms(1234567, 42, B, A)
    assert u2.min() > 0 and u2.max() < 1
    ref2 = orc.gumbel_argmax(logits, u2)
    g2 = -np.log(-np.log(u2)); s2 = np.sort(logits + g2, axis=1)
    bad2 = (act2.cpu().numpy() != ref2) & ((s2[:, -1] - s2[:, -2]) > 1e-4)
    assert not bad2.any()


def test_philox_known_answer():
    # Random123 known-answer test vectors for philox4x32-10
    z = orc.philox4x32_10(np.zeros((1, 4), np.uint32), np.zeros(2, np.uint32))[0]
    assert [hex(int(v)) for v in z] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]
    f = orc.philox4x32_10(np.full((1, 4), 0xFFFFFFFF, np.uint32), np.full(2, 0xFFFFFFFF, np.uint32))[0]
    assert [hex(int(v)) for v in f] == ["0x408f276d", "0x41c83b0e", "0xa20bc7c6", "0x6d5451fd"]


# ------------------------------------------------------------------------------------------- PPO loss
@pytest.mark.parametrize("B,A", [(320, 4), (256, 4), (4096, 4), (7, 2), (200, 18)])
def test_ppo_loss_grad_matches_autograd(xb, B, A):
    from xingtian_b200.engine import _ptr, stream_ptr
    rng = np.random.default_rng(B + A)
    logits = rng.standard_normal((B, A)).astype(np.float32)
    v = rng.standard_normal(B).astype(np.float32)
    action = rng.integers(0, A, B).astype(np.int32)
    old_logp = (np.log(1.0 / A) + 0.3 * rng.standard_normal(B)).astype(np.float32)
    adv = rng.standard_normal(B).astype(np.float32)
    old_v = (v + rng.standard_normal(B) * 4).astype(np.float32)
    target_v = rng.standard_normal(B).astype(np.float32)
    hp = xb["capi"].PpoHyper(0.1, 0.003, 5.0, 1.0)
    lt = torch.from_numpy(logits).requires_grad_(True); vt = torch.from_numpy(v).view(-1, 1).requires_grad_(True)
    c = lambda a: torch.from_numpy(a).view(-1, 1)
    loss = orc.ppo_loss(lt, vt, torch.from_numpy(action), c(old_logp), c(adv), c(old_v), c(target_v), 0.1, 0.003, 5.0, 1.0)
    loss.backward()
    dl = torch.empty(B, A, device="cuda"); dv = torch.empty(B, device="cuda"); lo = torch.zeros(1, device="cuda")
    xb["capi"].check(xb["lib"].xtb_ppo_loss_grad(_ptr(dev(logits)), _ptr(dev(v)), None, _ptr(dev(action)), _ptr(dev(old_logp)), _ptr(dev(adv)),
                                                _ptr(dev(old_v)), _ptr(dev(target_v)), B, A, C.byref(hp), 1.0 / B, _ptr(dl), _ptr(dv), _ptr(lo), stream_ptr()))
    assert abs(float(lo.cpu()[0]) - float(loss)) < REL * max(1.0, abs(float(loss)))
    assert rel_err(dl.cpu().numpy(), lt.grad.numpy()) < REL
    assert rel_err(dv.cpu().numpy(), vt.grad.numpy()[:, 0]) < REL


# ------------------------------------------------------------------------------------------- Adam
@pytest.mark.parametrize("mode", ["global", "per_tensor", "none"])
def test_adam_clip_ten_steps(xb, mode):
    from xingtian_b200.engine import _ptr, stream_ptr
    capi = xb["capi"]
    n = 847493 if mode == "global" else 50021
    rng = np.random.default_rng(5)
    p0 = rng.standard_normal(n).astype(np.float32) * 0.05
    seg = [0, 1000, 1032, 30000, n]
    p = dev(p0.copy()); m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    cm = {"global": capi.CLIP_GLOBAL_NORM, "per_tensor": capi.CLIP_PER_TENSOR, "none": capi.CLIP_NONE}[mode]
    clip = 5.0 if mode == "global" else 0.7
    eps = 1e-8 if mode == "global" else 1e-7
    h = C.c_void_p()
    segarr = (C.c_longlong * len(seg))(*seg)
    capi.check(xb["lib"].xtb_adam_create(n, 2.5e-4, 0.9, 0.999, eps, cm, clip, segarr, len(seg) - 1, _ptr(m), _ptr(v), C.byref(h)))
    ref_p = [torch.from_numpy(p0[seg[i]:seg[i + 1]].copy()) for i in range(len(seg) - 1)]
    opt = orc.TFAdam(ref_p, 2.5e-4, eps=eps)
    for step in range(10):
        g = (rng.standard_normal(n) * (0.02 if step % 2 else 0.002)).astype(np.float32)
        gl = [torch.from_numpy(g[seg[i]:seg[i + 1]].copy()) for i in range(len(seg) - 1)]
        if mode == "global":
            gl, gn = orc.clip_by_global_norm(gl, clip)
        elif mode == "per_tensor":
            gl = [x * (clip / float(x.norm())) if float(x.norm()) > clip else x for x in gl]
        opt.step(gl)
        capi.check(xb["lib"].xtb_adam_step(h, _ptr(p), _ptr(dev(g)), 1.0, stream_ptr()))
    ref = np.concatenate([x.numpy() for x in ref_p])
    assert rel_err(p.cpu().numpy() - p0, ref - p0) < REL      # compare the UPDATE, not the weights
    xb["lib"].xtb_adam_destroy(h)


def test_rmsprop_centered_ten_steps_and_lr_updates(xb):
    """a14: tf.train.RMSPropOptimizer(lr, decay=.99, epsilon=.1, centered=True) + clip_by_global_norm(40) on the flat bucket
    (impala_cnn_opt.py:205-215), and xtb_adam_set_lr between steps (the linear_cosine_decay schedule of :234-249)."""
    from xingtian_b200.engine import _ptr, stream_ptr
    capi = xb["capi"]
    n = 100003
    rng = np.random.default_rng(7)
    p0 = rng.standard_normal(n).astype(np.float32) * 0.05
    p = dev(p0.copy()); ms = torch.ones(n, device="cuda"); v = torch.zeros(n, device="cuda"); mg = torch.zeros(n, device="cuda")
    h = C.c_void_p()
    seg = (C.c_longlong * 2)(0, n)
    capi.check(xb["lib"].xtb_adam_create(n, 5e-4, 0.9, 0.999, 1e-8, capi.CLIP_GLOBAL_NORM, 40.0, seg, 1, _ptr(ms), _ptr(v), C.byref(h)))
    capi.check(xb["lib"].xtb_opt_use_rmsprop(h, _ptr(mg), 0.99, 0.1))
    ref_p = [torch.from_numpy(p0.copy())]
    opt = orc.TFRMSProp(ref_p, 5e-4, decay=0.99, eps=0.1)
    for step in range(10):
        lr = orc.linear_cosine_decay(5e-4, step * 1500, 20000.0, beta=1e-6 / 20000.0)
        opt.lr = lr
        capi.check(xb["lib"].xtb_adam_set_lr(h, lr))
        g = (rng.standard_normal(n) * (0.5 if step % 2 else 0.05)).astype(np.float32)      # |g| ~ 158 / 15.8: clip 40 bites on odd steps
        gl, _ = orc.clip_by_global_norm([torch.from_numpy(g.copy())], 40.0)
        opt.step(gl)
        capi.check(xb["lib"].xtb_adam_step(h, _ptr(p), _ptr(dev(g)), 1.0, stream_ptr()))
    assert rel_err(p.cpu().numpy() - p0, ref_p[0].numpy() - p0) < REL
    assert rel_err(ms.cpu().numpy(), opt.ms[0].numpy()) < REL and rel_err(mg.cpu().numpy(), opt.mg[0].numpy()) < REL
    xb["lib"].xtb_adam_destroy(h)


# ------------------------------------------------------------------------------------------- networks
def _arch_cases():
    return {
        "ppo_cnn": (orc.ppo_cnn_arch(), 847493),
        "ppo_cnn_sep": (orc.ppo_cnn_arch(hidden_sizes=(64,), vf_share_layers=False), None),
        "ppo_mlp": (orc.ppo_mlp_arch(), None),
        "ppo_mlp_shared": (orc.ppo_mlp_arch(vf_share_layers=True), None),
        "impala_cnn": (orc.impala_cnn_arch(), 1005109),
        "dqn_cnn": (orc.dqn_cnn_arch(), 882084),
        "dqn_mlp": (orc.dqn_mlp_arch(), None),
    }


@pytest.fixture(params=[1, 0], ids=["tcgen05", "fp32"])
def tc_mode(request, xb):
    lib = xb["lib"]
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(request.param)
    yield request.param
    lib.xtb_set_tc_mode(old)


def l2_rel(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _smooth(arch):
    """Same layers with relu -> tanh: gradients become smooth in the forward rounding, so every kernel
    (gathers, GEMMs, masks) can be held to the max-norm 1e-3 contract."""
    layers = [(n, k, s, dict(sp, act=("tanh" if sp.get("act") == "relu" else sp.get("act")))) for n, k, s, sp in arch["layers"]]
    return dict(arch, layers=layers)


@pytest.mark.parametrize("smooth", [True, False], ids=["tanh", "relu"])
@pytest.mark.parametrize("case,B", [("ppo_cnn", 5), ("ppo_cnn", 64), ("ppo_cnn", 320), ("ppo_cnn_sep", 9), ("ppo_mlp", 200), ("ppo_mlp_shared", 33),
                                    ("impala_cnn", 6), ("impala_cnn", 130), ("dqn_cnn", 7), ("dqn_cnn", 129), ("dqn_mlp", 32)])
def test_network_forward_backward(xb, tc_mode, case, B, smooth):
    """a1-a5: forward of every tensor and the full parameter gradient vs torch-CPU autograd, on the
    tcgen05 path and on the fp32 CUDA-core path.

    ReLU makes the gradient a discontinuous function of the forward rounding: a unit whose
    pre-activation is within rounding error of zero (bf16x3: ~1e-5 relative; expected count grows
    with B) takes the other branch than in the reference and its whole receptive field changes.  So
    the max-norm 1e-3 contract is asserted on the tanh variant of every network (identical kernels),
    and the ReLU networks are held to 1e-3 on the forward tensors and to a norm-wise bound on the
    gradients."""
    from xingtian_b200.engine import Net
    arch, nparam = _arch_cases()[case]
    if smooth:
        arch = _smooth(arch)
    w = orc.init_weights(arch, seed=11)
    for k in w:                                   # non-zero biases so bias grads/paths are exercised
        if k.endswith("/bias"):
            w[k] = (np.random.default_rng(1).standard_normal(w[k].shape) * 0.05).astype(np.float32)
    net = Net(arch, max_batch=max(B, 8))
    if nparam:
        assert net.n_params == nparam
    assert list(net.ptable.keys()) == list(orc.param_shapes(arch).keys())
    net.set_weights(w)
    rng = np.random.default_rng(2)
    nrows = B + 3
    if arch["input_dtype"] == "uint8":
        obs = rng.integers(0, 256, (nrows,) + arch["state_dim"], dtype=np.uint8)
    else:
        obs = rng.standard_normal((nrows,) + arch["state_dim"]).astype(np.float32)
    idx = rng.permutation(nrows)[:B].astype(np.int32)
    obs_d, idx_d = dev(obs), dev(idx)
    net.forward(obs_d, B, idx=idx_d)
    params = {k: torch.from_numpy(v.copy()).requires_grad_(True) for k, v in w.items()}
    ref = orc.forward(arch, params, obs[idx], keep=True)
    for name, _, _, _ in arch["layers"]:
        got = net.tensor(name)[:B].cpu().numpy()
        assert rel_err(got, ref[name].detach().reshape(B, -1).numpy()) < REL, name
    # backward with random head gradients
    heads = arch["outputs"]
    loss = 0
    for h in heads:
        gh = rng.standard_normal(tuple(ref[h].shape)).astype(np.float32)
        net.tensor_grad(h)[:B].copy_(dev(gh.reshape(B, -1)))
        loss = loss + (ref[h] * torch.from_numpy(gh)).sum()
    loss.backward()
    net.backward(obs_d, B, heads, idx=idx_d)
    got = net.get_weights(net.grads)
    if smooth:
        errs = {k: rel_err(got[k], params[k].grad.numpy()) for k in w}
        bad = {k: "%.2e" % e for k, e in errs.items() if not e < REL}
    else:
        errs = {k: l2_rel(got[k], params[k].grad.numpy()) for k in w}
        # mask flips (see the float64 test below); their relative weight grows as the batch shrinks: 1.5e-2 at B=64
        bad = {k: "%.2e" % e for k, e in errs.items() if not e < 3e-2}
    assert not bad, bad
    # round trip of the weight dict
    back = net.get_weights()
    for k in w:
        np.testing.assert_array_equal(back[k], w[k])


from parity_record import record as _record  # noqa: E402


@pytest.mark.parametrize("smooth", [True, False], ids=["tanh", "relu"])
@pytest.mark.parametrize("case,B", [("ppo_cnn", 320), ("ppo_cnn", 4096), ("impala_cnn", 130), ("impala_cnn", 512), ("dqn_cnn", 129),
                                    ("dqn_cnn", 512)])          # C2 / C5 / C3 / C4 minibatch sizes and ragged ones
def test_gradient_distance_to_float64_vs_torch_cpu(xb, tc_mode, case, B, smooth):
    """Round-1 verdict item 4: the float64 restatement (oracle precision("f64"), pinned by tests/test_oracle_f64.py) is the
    yardstick; e_gpu = |gpu - f64| and e_cpu = |torch-CPU fp32 - f64|, forward tensors in max-norm and parameter gradients
    in relative L2, at config batch sizes.

    tanh variant (smooth: every kernel, no kinks): the fp32 CUDA-core path must be as close to exact arithmetic as the
    reference's own fp32 run, e_gpu <= 2 e_cpu + 2e-6; the tensor-core path carries 16-bit operand mantissas (bf16 hi + lo, the
    lo*lo term dropped: ~2^-17 per operand against 2^-24) and is held to TC_FWD_BOUND / TC_GRAD_BOUND,
    two orders inside the 1e-3 parity target.
    ReLU networks: one unit whose pre-activation lies within the forward rounding error of zero takes the other branch and
    moves the conv gradients by ~5e-4 in L2 -- observed on an H100 for the GPU fp32 path on dqn_cnn (5.9e-4 against the CPU's
    1.2e-6) and, the other way round, for torch-CPU fp32 on impala_cnn (CPU 6.0e-4, GPU 2.9e-7); with the 1e-5 forward error
    of bf16x3 a handful flip at B=320 (2.6e-3).  Hence the flip allowances RELU_FLIP_*.  All observed errors are recorded
    through tests/parity_record.py."""
    from xingtian_b200.engine import Net
    arch, _ = _arch_cases()[case]
    if smooth:
        arch = _smooth(arch)
    w = orc.init_weights(arch, seed=11)
    for k in w:
        if k.endswith("/bias"):
            w[k] = (np.random.default_rng(1).standard_normal(w[k].shape) * 0.05).astype(np.float32)
    net = Net(arch, max_batch=B)
    net.set_weights(w)
    rng = np.random.default_rng(2)
    obs = rng.integers(0, 256, (B,) + arch["state_dim"], dtype=np.uint8)
    heads = arch["outputs"]
    gh = {h: rng.standard_normal((B, int(np.prod(orc.tensor_shapes(arch)[h])))).astype(np.float32) for h in heads}

    def cpu(prec):
        with orc.precision(prec):
            params = {k: torch.from_numpy(v.astype(np.float64 if prec == "f64" else np.float32)).requires_grad_(True) for k, v in w.items()}
            t = orc.forward(arch, params, obs, keep=True)
            loss = sum((t[h].reshape(B, -1) * torch.from_numpy(gh[h]).to(t[h].dtype)).sum() for h in heads)
            loss.backward()
            return ({n: t[n].detach().reshape(B, -1).numpy() for n, _, _, _ in arch["layers"]},
                    {k: params[k].grad.numpy() for k in w})
    f64_t, f64_g = cpu("f64")
    f32_t, f32_g = cpu("f32")
    obs_d = dev(obs)
    net.forward(obs_d, B)
    for h in heads:
        net.tensor_grad(h)[:B].copy_(dev(gh[h]))
    gpu_t = {n: net.tensor(n)[:B].cpu().numpy() for n, _, _, _ in arch["layers"]}
    net.backward(obs_d, B, heads)
    gpu_g = net.get_weights(net.grads)
    fwd = {n: (rel_err(gpu_t[n], f64_t[n]), rel_err(f32_t[n], f64_t[n])) for n in gpu_t}
    grd = {k: (l2_rel(gpu_g[k], f64_g[k]), l2_rel(f32_g[k], f64_g[k])) for k in w}
    _record("grad_vs_f64/%s/B%d/%s/%s" % (case, B, "tanh" if smooth else "relu", "tcgen05" if tc_mode else "fp32"),
            {"forward_max_rel(gpu,cpu32)": {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in fwd.items()},
             "grad_l2_rel(gpu,cpu32)": {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in grd.items()}})
    flip = 0.0 if smooth else (RELU_FLIP_TC if tc_mode else RELU_FLIP_F32)
    if tc_mode:
        bad = {k: v for k, v in fwd.items() if not v[0] < TC_FWD_BOUND}
        bad.update({k: v for k, v in grd.items() if not v[0] < TC_GRAD_BOUND + flip})
    else:
        bad = {k: v for k, v in fwd.items() if not v[0] <= 2 * v[1] + F32_FLOOR}
        bad.update({k: v for k, v in grd.items() if not v[0] <= 2 * v[1] + F32_FLOOR + flip})
    assert not bad, bad


F32_FLOOR = 2e-6          # a few fp32 ulps of summation-order slack on top of 2 x the CPU's own error
TC_FWD_BOUND = 5e-5       # bf16x3 forward, max-norm relative to float64 (observed <= 1.3e-5)
TC_GRAD_BOUND = 6e-5      # bf16x3 parameter gradients without kinks, relative L2 (observed <= 1.5e-5)
RELU_FLIP_F32 = 4e-3      # ReLU mask flips at fp32 forward error (observed 5.9e-4 at B=129, 1.7e-3 at B=4096 where torch-CPU has 1.4e-3)
RELU_FLIP_TC = 2e-2       # ... at bf16x3 forward error (observed 2.6e-3 at B=320, 8.4e-3 at B=4096; torch-CPU fp32 itself: 1.4e-3)
