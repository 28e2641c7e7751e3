"""The optimiser step that ends every training step (csrc/optim.cuh: sqnorm_kernel, then adam_kernel or rmsprop_kernel)
against float64, and the weight-blob refresh those kernels perform, bit for bit against bp_wprep_kernel.

Step: the oracle's tf.train.Adam (through its Keras restatement, KerasAdam, for per-tensor clipnorm
and `decay`) and centred RMSProp, with clip_by_global_norm, under precision("f64") as the yardstick and precision("f32")
as the torch-CPU fp32 reference.  grad_scale multiplies the gradient before clipping (include/xtb200.h).  Segment layouts
reach the optimiser's scalar paths: chunks that start off a multiple of 4 elements, 1..7-element tensors several to one
sqnorm block, empty tensors, odd tails; and the per-tensor layouts of the products.  Every segment's gradient has its own
norm, spread over decades, so that per-tensor clipping bites on some tensors and not on others and global clipping bites
on odd steps only; one tensor is all zeros and one has |g| ~ eps.  Bounds, as in
test_gradient_distance_to_float64_vs_torch_cpu: the update p - p0 and the optimiser state within REL (max-norm relative)
of float64 and, in relative L2, at most 2x torch-CPU fp32's own distance + F32_FLOOR.  The device's pre-clip global norm
(fp32 partial sums of at most SQN_GROUP * OPT_CHUNK = 4096 squares per block, fp64 atomics across blocks, so a few fp32
ulps) within NORM_BOUND of float64.

Blobs: the step rewrites the bf16 hi/lo weight blobs of the tensor-core layers from the fp32 parameters it produced.
xtb_net_sync_weights (bp_wprep_kernel, its own index map) rewrites exactly that region from the same parameters, so the
workspace must not change by a single bit when it runs after a step."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from parity_record import record as _record
from test_gpu_kernels import F32_FLOOR, REL, _keepalive, dev, l2_rel, rel_err, xb  # noqa: F401
from test_gpu_layer_sweep import CASES

pytestmark = pytest.mark.gpu

# Relative; from the summation error estimate above, not from a device measurement.  Observed <= 1.0e-7 on an H100 80GB
# HBM3 at a 400 W power limit, where the step's update stayed within max-rel 4.1e-5 of float64 and its relative L2
# distance never exceeded twice torch-CPU fp32's by more than 1e-7.
NORM_BOUND = 1e-5
STEPS = 12


def f32(x):
    """The float the C-ABI receives.  The yardstick computes with the hyperparameters the device was given: 1 - 0.999 in
    float64 is 1.3e-5 away from 1 - float32(0.999), which the device (like TF on its fp32 slots) computes exactly."""
    return float(np.float32(x))


LR, BETA1, BETA2, ADAM_EPS, RMS_RHO, RMS_EPS = (f32(x) for x in (1e-3, 0.9, 0.999, 1e-8, 0.99, 0.1))
DECAY = f32(0.05)        # Keras `decay`, large enough to move lr by several percent over the run
EXPS = [2.0, -3.0, 0.5, -1.0, 1.0, -2.0, 0.3, -0.5, 1.5, -1.5]   # log10 of the per-segment gradient norms
JITTER = (0.8, 1.25)     # with step factors 3 and 1/3, no segment norm comes within 15% of the per-tensor clip 1.0


def _offsets(shapes):
    return [0] + [int(x) for x in np.cumsum([int(np.prod(s)) for s in shapes.values()])]


SYNTH = {
    "n1": [0, 1],
    "n5": [0, 5],
    "mixed": [0, 1, 3, 4, 9, 1033, 2057, 6154],                           # lengths 1, 2, 1, 5, 1024, 1024, 4097
    "many_short": [0] + [int(x) for x in np.cumsum([1 + i % 7 for i in range(64)])],
    "empty_segments": [0, 0, 7, 7, 7, 1031, 2050, 2050],
    "long_at_1_mod_4": [0, 1, 4098, 4103],
}
REAL = {
    "ppo_mlp": lambda: _offsets(orc.param_shapes(orc.ppo_mlp_arch())),
    "ppo_cnn": lambda: _offsets(orc.param_shapes(orc.ppo_cnn_arch())),
    "impala_cnn": lambda: _offsets(orc.param_shapes(orc.impala_cnn_arch())),
    "dqn_cnn_dueling": lambda: _offsets(orc.param_shapes(orc.dqn_cnn_arch(dueling=True))),
}
BIG = {"ppo_cnn": 847493, "impala_cnn": 1005109, "dqn_cnn_dueling": 882341}
BIG_ROWS = {("adam", "global"), ("adam", "per_tensor"), ("rmsprop", "global")}   # what the products run


def _layout(name):
    return list(SYNTH[name]) if name in SYNTH else REAL[name]()


def _rows():
    rows = []
    for layout in list(SYNTH) + list(REAL):
        for opt in ("adam", "rmsprop"):
            for mode in ("none", "global", "per_tensor"):
                if layout in BIG and (opt, mode) not in BIG_ROWS:
                    continue
                for gs in (1.0, 0.5, -0.5):
                    rows.append(pytest.param(layout, opt, mode, gs, id="%s-%s-%s-gs%g" % (layout, opt, mode, gs)))
    return rows


def _schedule(opt, gs):
    """(learning rates, Keras decay): grad_scale 1 keeps lr constant, 0.5 sets it before every step, -0.5 sets it for
    RMSProp (IMPALA's schedule) and uses `decay` for Adam"""
    if gs == 1.0:
        return [LR] * STEPS, 0.0
    if gs == -0.5 and opt == "adam":
        return [LR] * STEPS, DECAY
    return [f32(LR * (1.0 - 0.06 * t)) for t in range(STEPS)], 0.0


def _gradients(offs, gs, eps, seed):
    """STEPS gradients and the global clip threshold.  Segment i has norm 10^EXPS[i] * jitter * f / |gs| with f = 3 on
    odd steps and 1/3 on even ones, so that grad_scale * g has the same norms for every grad_scale; with four or more
    non-empty segments the second is all zeros and the third has |g| ~ eps."""
    rng = np.random.default_rng(seed)
    live = [s for s in range(len(offs) - 1) if offs[s + 1] > offs[s]]
    zero, tiny = (live[1], live[2]) if len(live) >= 4 else (None, None)
    base = [10.0 ** EXPS[i % len(EXPS)] for i, s in enumerate(live) if s not in (zero, tiny)]
    clip_global = f32(np.sqrt(np.sum(np.square(base))))        # scaled global norm: >= 2.4x it on odd steps, <= 0.42x on even
    out = []
    for t in range(STEPS):
        f = 3.0 if t % 2 else 1.0 / 3.0
        g = np.zeros(offs[-1], np.float64)
        for i, s in enumerate(live):
            a, b = offs[s], offs[s + 1]
            x = rng.standard_normal(b - a)
            if s == zero:
                continue
            if s == tiny:
                g[a:b] = x * eps
                continue
            g[a:b] = x / np.linalg.norm(x) * 10.0 ** EXPS[i % len(EXPS)] * JITTER[rng.integers(2)] * f / abs(gs)
        out.append(g.astype(np.float32))
    return out, clip_global


def _reference(offs, opt, mode, clip, gs, grads, lrs, decay, p0, prec):
    """parameters, optimiser state and pre-clip global norms of the oracle in `prec`"""
    dt = torch.float64 if prec == "f64" else torch.float32
    segs = list(zip(offs[:-1], offs[1:]))
    with orc.precision(prec):
        ps = [torch.from_numpy(p0[a:b]).to(dt).clone() for a, b in segs]     # updated in place: never alias p0
        if opt == "adam":
            o = orc.KerasAdam(ps, LR, clipnorm=clip if mode == "per_tensor" else None, decay=decay, eps=ADAM_EPS)
            o.b1, o.b2 = BETA1, BETA2
        else:
            o = orc.TFRMSProp(ps, LR, decay=RMS_RHO, eps=RMS_EPS)
        norms = []
        for g, lr in zip(grads, lrs):
            gl = [torch.from_numpy(g[a:b]).to(dt) * gs for a, b in segs]
            norms.append(float(np.sqrt(sum(float(x.double().pow(2).sum()) for x in gl))))
            if mode == "global":
                gl, _ = orc.clip_by_global_norm(gl, clip)
            elif mode == "per_tensor" and opt == "rmsprop":
                gl = orc.clip_per_tensor(gl, clip)            # (KerasAdam clips per tensor itself)
            if opt == "adam":
                o.base_lr = lr
            else:
                o.lr = lr
            o.step(gl)
    cat = lambda ts: np.concatenate([t.numpy().astype(np.float64) for t in ts])   # noqa: E731
    state = {"m": cat(o.m), "v": cat(o.v)} if opt == "adam" else {"ms": cat(o.ms), "mg": cat(o.mg)}
    return cat(ps), state, np.array(norms)


def _grad_norm(lib, capi, h):
    from xingtian_b200.engine import stream_ptr
    out = torch.empty(1, dtype=torch.float32)
    torch.cuda.synchronize()
    capi.check(lib.xtb_copy_d2h(C.c_void_p(out.data_ptr()), C.c_void_p(lib.xtb_adam_grad_norm(h)), 4, stream_ptr()))
    torch.cuda.synchronize()
    return float(out[0])


MODES = {"none": 0, "global": 1, "per_tensor": 2}


def _device(xb, offs, opt, mode, clip, gs, grads, lrs, decay, p0, set_lr):
    """the same run through xtb_adam_create / xtb_adam_step"""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib, capi = xb["lib"], xb["capi"]
    n = offs[-1]
    p = dev(p0.copy())
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    seg = (C.c_longlong * len(offs))(*offs)
    h = C.c_void_p()
    capi.check(lib.xtb_adam_create(n, LR, BETA1, BETA2, ADAM_EPS, MODES[mode], clip, seg, len(offs) - 1, _ptr(m), _ptr(v),
                                   C.byref(h)))
    try:
        if opt == "rmsprop":
            mg = torch.zeros(n, device="cuda")
            capi.check(lib.xtb_opt_use_rmsprop(h, _ptr(mg), RMS_RHO, RMS_EPS))
        if decay:
            capi.check(lib.xtb_adam_set_decay(h, decay))
        norms = []
        for g, lr in zip(grads, lrs):
            if set_lr:
                capi.check(lib.xtb_adam_set_lr(h, lr))
            capi.check(lib.xtb_adam_step(h, _ptr(p), _ptr(dev(g)), gs, stream_ptr()))
            norms.append(_grad_norm(lib, capi, h))
        torch.cuda.synchronize()
        to64 = lambda t: t.cpu().numpy().astype(np.float64)   # noqa: E731
        state = {"m": to64(m), "v": to64(v)} if opt == "adam" else {"ms": to64(m), "mg": to64(mg)}
        return to64(p), state, np.array(norms)
    finally:
        lib.xtb_adam_destroy(h)


# ------------------------------------------------------------------------------------------- the step against float64
@pytest.mark.parametrize("layout,opt,mode,gs", _rows())
def test_step_against_float64(xb, layout, opt, mode, gs):
    offs = _layout(layout)
    if layout in BIG:
        assert offs[-1] == BIG[layout]
    eps = ADAM_EPS if opt == "adam" else RMS_EPS
    grads, clip_global = _gradients(offs, gs, eps, seed=len(offs) * 7 + offs[-1])
    clip = {"none": 0.0, "global": clip_global, "per_tensor": 1.0}[mode]
    lrs, decay = _schedule(opt, gs)
    set_lr = any(lr != LR for lr in lrs)
    p0 = (np.random.default_rng(3).standard_normal(offs[-1]) * 0.05).astype(np.float32)
    p_gpu, s_gpu, n_gpu = _device(xb, offs, opt, mode, clip, gs, grads, lrs, decay, p0, set_lr)
    p64, s64, n64 = _reference(offs, opt, mode, clip, gs, grads, lrs, decay, p0, "f64")
    p32, s32, _ = _reference(offs, opt, mode, clip, gs, grads, lrs, decay, p0, "f32")
    base = p0.astype(np.float64)
    got = {"update": p_gpu - base, **s_gpu}
    ref = {"update": p64 - base, **s64}
    cpu = {"update": p32 - base, **s32}
    dist = {k: (rel_err(got[k], ref[k]), l2_rel(got[k], ref[k]), l2_rel(cpu[k], ref[k])) for k in got}
    norm_err = float(np.max(np.abs(n_gpu - n64) / n64))
    _record("optim/%s/%s/%s/gs%g" % (layout, opt, mode, gs),
            {"max_rel,l2_rel(gpu),l2_rel(cpu32)": {k: ["%.2e" % x for x in d] for k, d in dist.items()},
             "grad_norm_rel": "%.2e" % norm_err})
    bad = {k: d for k, d in dist.items() if not (d[0] < REL and d[1] <= 2 * d[2] + F32_FLOOR)}
    assert not bad, bad
    assert norm_err < NORM_BOUND, (norm_err, n_gpu, n64)
    if mode == "global":                                     # the data exercised both sides of the clip
        scaled = n64 / clip
        assert (scaled[1::2] > 2).all() and (scaled[0::2] < 0.5).all(), scaled


# ------------------------------------------------------------------------------------------- argument checks on a live optimiser
def test_empty_segment_is_a_zero_norm_tensor(xb):
    """Equal neighbouring offsets are accepted: the step is bitwise the step of the layout without the empty tensors."""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib, capi = xb["lib"], xb["capi"]
    rng = np.random.default_rng(21)
    p0 = (rng.standard_normal(9) * 0.05).astype(np.float32)
    grads = [(rng.standard_normal(9) * 3).astype(np.float32) for _ in range(4)]
    out = []
    for offs in ([0, 0, 5, 5, 9, 9], [0, 5, 9]):
        p, m, v = dev(p0.copy()), torch.zeros(9, device="cuda"), torch.zeros(9, device="cuda")
        seg = (C.c_longlong * len(offs))(*offs)
        h = C.c_void_p()
        capi.check(lib.xtb_adam_create(9, LR, BETA1, BETA2, 1e-7, MODES["per_tensor"], 1.0, seg, len(offs) - 1, _ptr(m), _ptr(v),
                                       C.byref(h)))
        norms = []
        for g in grads:
            capi.check(lib.xtb_adam_step(h, _ptr(p), _ptr(dev(g)), 1.0, stream_ptr()))
            norms.append(_grad_norm(lib, capi, h))
        lib.xtb_adam_destroy(h)
        out.append((p.cpu(), m.cpu(), v.cpu(), norms))
    (pa, ma, va, na), (pb, mb, vb, nb) = out
    assert torch.equal(pa, pb) and torch.equal(ma, mb) and torch.equal(va, vb) and na == nb
    assert not torch.equal(pa, torch.from_numpy(p0))


def test_step_rejects_misaligned_buffers_and_launches_nothing(xb):
    """params / grads 4 bytes off a 16-byte boundary (a torch view such as flat[1:]): XTB_ERR_ARG, no launch, params
    untouched; a misaligned RMSProp mean-gradient slot is refused the same way."""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib, capi = xb["lib"], xb["capi"]
    n = 4099
    p = torch.randn(n + 4, device="cuda")
    g = torch.randn(n + 4, device="cuda")
    m, v, mg = torch.zeros(n + 4, device="cuda"), torch.zeros(n + 4, device="cuda"), torch.zeros(n + 4, device="cuda")
    seg = (C.c_longlong * 2)(0, n)
    h = C.c_void_p()
    capi.check(lib.xtb_adam_create(n, LR, BETA1, BETA2, ADAM_EPS, MODES["global"], 1.0, seg, 1, _ptr(m), _ptr(v), C.byref(h)))
    try:
        torch.cuda.synchronize()
        p_before = p.clone()
        for pp, gg in ((p[1:], g), (p, g[1:]), (p[3:], g[1:])):
            launches = lib.xtb_launch_count()
            assert lib.xtb_adam_step(h, _ptr(pp), _ptr(gg), 1.0, stream_ptr()) == -1
            assert b"16-byte aligned" in lib.xtb_last_error()
            assert lib.xtb_launch_count() == launches
        assert lib.xtb_opt_use_rmsprop(h, _ptr(mg[1:]), RMS_RHO, RMS_EPS) == -1
        assert b"16-byte aligned" in lib.xtb_last_error()
        torch.cuda.synchronize()
        assert torch.equal(p, p_before)
        capi.check(lib.xtb_adam_step(h, _ptr(p), _ptr(g), 1.0, stream_ptr()))     # still a working optimiser
        torch.cuda.synchronize()
        assert not torch.equal(p, p_before)
    finally:
        lib.xtb_adam_destroy(h)


# ------------------------------------------------------------------------------------------- weight blobs, bit for bit
def _blob_nets():
    nets = {"sweep_" + case: (lambda make=make: make("tanh"), max_batch)
            for case, (make, B, max_batch, gather, expect) in CASES.items()}
    nets["ppo_cnn"] = (orc.ppo_cnn_arch, 64)
    nets["impala_cnn"] = (orc.impala_cnn_arch, 64)
    nets["dqn_cnn_dueling"] = (lambda: orc.dqn_cnn_arch(dueling=True), 64)
    return nets


BLOB_NETS = _blob_nets()
BLOB_OPTS = [("adam", "global"), ("adam", "per_tensor"), ("rmsprop", "global")]


@pytest.mark.parametrize("name", list(BLOB_NETS))
def test_step_refreshes_weight_blobs_as_sync_weights_does(xb, name):
    from xingtian_b200.engine import Adam, Net
    make, max_batch = BLOB_NETS[name]
    arch = make()
    net = Net(arch, max_batch=max_batch)
    tc = [l[0] for i, l in enumerate(arch["layers"]) if net.layer_plan(i)["tc"]]
    assert tc, "no tensor-core layer: no weight blob to check"
    rng = np.random.default_rng(17)
    for opt_name, mode in BLOB_OPTS:
        net.set_weights({k: (rng.standard_normal(shape) * 0.05).astype(np.float32) for k, (_, shape) in net.ptable.items()})
        opt = Adam(net, LR, clip_mode=MODES[mode], clip=1.0)
        if opt_name == "rmsprop":
            opt.use_rmsprop(RMS_RHO, RMS_EPS)
        for step in range(3):
            net.grads.copy_(torch.from_numpy(rng.standard_normal(net.n_params).astype(np.float32)))
            before = net.ws.clone()
            opt.step()
            after = net.ws.clone()
            net.params_changed()                   # bp_wprep_kernel from the same fp32 parameters
            diff = int((net.ws != after).sum())
            assert diff == 0, (opt_name, mode, step, tc, diff)
            assert not torch.equal(before, after), (opt_name, mode, step)
        del opt
