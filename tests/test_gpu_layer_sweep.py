"""The layer engine across the conv and dense geometries xtb_net_create accepts, on the tensor-core (wgmma) path and on
the fp32 CUDA-core path, against the float64 restatement of the oracle.

Each case is a small network.  A layer that reads the observation runs on the tensor cores only as a space-to-depth
("s2d") first layer, so a conv under test is fed by an s2d stem: uint8 frames (4H, 4W, 4), conv k=4 s=4 VALID with
Cout = the Cin under test (itself a tensor-core layer with R = 1).  Every case asserts through Net.layer_plan that its
layers were planned onto the path the case was written for, and test_sweep_covers_the_tensor_core_plan keeps the table
from losing coverage.

Forward: every tensor against oracle.forward under precision("f64").  Backward: random head gradients G (d/d pre-
activation, include/xtb200.h), reference loss sum_h pre_h . G_h, every weight and bias gradient.  ReLU: the float64
backward runs through pre * mask with the mask of the GPU forward (out > 0), after asserting that this mask differs from
the float64 sign only where |pre| < 1e-4 max|pre|; branch flips are then out of the comparison and ReLU cases carry the
same bounds as tanh ones.  Bounds are those of test_gradient_distance_to_float64_vs_torch_cpu: tensor-core path forward
max-rel < TC_FWD_BOUND, gradients L2-rel < TC_GRAD_BOUND and max-rel < 1e-3; fp32 path at most 2x torch-CPU fp32's
own distance from float64 + F32_FLOOR."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import xt_oracle as orc
from parity_record import record as _record
from test_gpu_kernels import (F32_FLOOR, REL, TC_FWD_BOUND, TC_GRAD_BOUND, _keepalive, dev, l2_rel, rel_err,  # noqa: F401
                              tc_mode, xb)

pytestmark = pytest.mark.gpu

MASK_TIE = 1e-4     # a GPU ReLU mask may differ from the float64 sign only where |pre| < MASK_TIE * max|pre|


# ------------------------------------------------------------------------------------------- networks of the sweep
def _conv(name, src, k, s, cout, pad, act):
    return (name, "conv", src, dict(k=k, s=s, cout=cout, pad=pad, act=act))


def _dense(name, src, n, act):
    return (name, "dense", src, dict(n=n, act=act))


def _stemmed(hw, cin, act, layers, outputs):
    """uint8 frames (4H, 4W, 4) -> s2d stem "x" (conv k4 s4 VALID) = an H x W x cin map -> `layers`"""
    h, w = hw
    return dict(input_dtype="uint8", state_dim=(4 * h, 4 * w, 4), scale=1.0 / 255.0,
                layers=[_conv("x", "obs", 4, 4, cin, "valid", act)] + layers, outputs=outputs)


def _one_conv(hw, cin, cout, k, s, pad):
    return lambda a: _stemmed(hw, cin, a, [_conv("y", "x", k, s, cout, pad, a)], ["y"])


def _s2d(hw, k, pad, cout):
    """the s2d first layer itself, read by a tensor-core conv head"""
    return lambda a: dict(input_dtype="uint8", state_dim=hw + (4,), scale=1.0 / 255.0,
                          layers=[_conv("y", "obs", k, 4, cout, pad, a), _conv("z", "y", 3, 2, 16, "valid", a)], outputs=["z"])


def _dense_pair(K, N):
    """float observations -> dense K (fp32: it reads the observation) -> tensor-core dense N"""
    return lambda a: dict(input_dtype="float32", state_dim=(20,), scale=1.0,
                          layers=[_dense("x", "obs", K, a), _dense("y", "x", N, a)], outputs=["y"])


def _dense_4096(N):
    """s2d stem 16 x 16 x 16 = 4096 features -> tensor-core dense N (split-K forward)"""
    return lambda a: _stemmed((16, 16), 16, a, [_dense("y", "x", N, a)], ["y"])


TC, F32 = dict(tc=True), dict(tc=False)

# name: (arch(act), B, max_batch, gather, {layer: expected layer_plan fields})
CASES = {
    # input pixels no filter tap reaches: the data gradient's `empty` select; N = 48 conv forward / weight gradient
    "empty_10x10_32to48_k3s2_valid": (_one_conv((10, 10), 32, 48, 3, 2, "valid"), 65, 65, False,
                                      {"x": dict(tc=True, s2d=True, R=1), "y": dict(tc=True, n_fwd=48, n_dg=32, dg_empty_units=19)}),
    "empty_9x9_32to32_k2s2_valid": (_one_conv((9, 9), 32, 32, 2, 2, "valid"), 129, 129, True,
                                    {"y": dict(tc=True, n_fwd=32, n_dg=32, dg_empty_units=17)}),
    # accumulator widths 16 / 48 / 64 on forward, data gradient and weight gradient; stride 4 after the stem
    "width_10x10_16to48_k3s1_same": (_one_conv((10, 10), 16, 48, 3, 1, "same"), 63, 100, False,
                                     {"y": dict(tc=True, n_fwd=48, n_dg=16, w_res=True, dg_empty_units=0)}),
    "width_12x12_48to16_k4s4_valid": (_one_conv((12, 12), 48, 16, 4, 4, "valid"), 64, 64, True,
                                      {"x": dict(tc=True, n_fwd=48), "y": dict(tc=True, n_fwd=16, n_dg=48)}),
    "width_6x6_64to64_k3s1_same": (_one_conv((6, 6), 64, 64, 3, 1, "same"), 200, 256, False,
                                   {"y": dict(tc=True, n_fwd=64, n_dg=64, w_res=False)}),
    # non-square map with asymmetric SAME padding; 5x5 SAME with streamed weights; 1x1 filter
    "odd_12x7_16to64_k3s2_same": (_one_conv((12, 7), 16, 64, 3, 2, "same"), 1, 40, False,
                                  {"y": dict(tc=True, n_fwd=64, n_dg=16)}),
    "odd_11x11_64to16_k5s1_same": (_one_conv((11, 11), 64, 16, 5, 1, "same"), 65, 65, False,
                                   {"y": dict(tc=True, n_fwd=16, n_dg=64, w_res=False, R=15)}),
    "odd_9x9_16to32_k1s1_valid": (_one_conv((9, 9), 16, 32, 1, 1, "valid"), 129, 129, True,
                                  {"y": dict(tc=True, n_fwd=32, n_dg=16, R=1)}),
    # the largest accepted weight-gradient grids
    "rlimit_8x8_64to16_k7s1_same": (_one_conv((8, 8), 64, 16, 7, 1, "same"), 64, 64, False,
                                    {"y": dict(tc=True, R=28, w_res=False)}),
    "rlimit_9x9_64to16_k8s1_valid": (_one_conv((9, 9), 64, 16, 8, 1, "valid"), 63, 63, True,
                                     {"y": dict(tc=True, R=32)}),
    # s2d first layers: k = 4 / 8 / 12, VALID and SAME, and an odd top padding (86 rows, SAME: padT = 3)
    "s2d_84x84_k4_valid": (_s2d((84, 84), 4, "valid", 16), 65, 65, False, {"y": dict(tc=True, s2d=True), "z": TC}),
    "s2d_84x84_k4_same": (_s2d((84, 84), 4, "same", 32), 1, 16, True, {"y": dict(tc=True, s2d=True), "z": TC}),
    "s2d_84x84_k8_valid": (_s2d((84, 84), 8, "valid", 32), 65, 65, True, {"y": dict(tc=True, s2d=True), "z": TC}),
    "s2d_84x84_k8_same": (_s2d((84, 84), 8, "same", 16), 129, 129, False, {"y": dict(tc=True, s2d=True), "z": TC}),
    "s2d_84x84_k12_valid": (_s2d((84, 84), 12, "valid", 48), 63, 63, False, {"y": dict(tc=True, s2d=True, n_fwd=48), "z": TC}),
    "s2d_84x84_k12_same": (_s2d((84, 84), 12, "same", 16), 64, 100, True, {"y": dict(tc=True, s2d=True), "z": TC}),
    "s2d_86x84_k8_same": (_s2d((86, 84), 8, "same", 32), 65, 65, True, {"y": dict(tc=True, s2d=True), "z": TC}),
    # one tensor read by two layers: the data-gradient `accumulate` epilogue and the gradient representation changes
    "dag_two_tc_convs": (lambda a: _stemmed((8, 8), 32, a, [
        _conv("y", "x", 3, 1, 32, "same", a), _conv("z1", "y", 3, 2, 16, "valid", a), _conv("z2", "y", 1, 1, 48, "valid", a)],
        ["z1", "z2"]), 65, 65, False, {"y": TC, "z1": TC, "z2": TC}),
    "dag_fp32_then_tc": (lambda a: _stemmed((8, 8), 32, a, [
        _conv("y", "x", 3, 1, 32, "same", a), _conv("z1", "y", 3, 1, 32, "same", a), _conv("z2", "y", 1, 2, 16, "valid", a)],
        ["z1", "z2"]), 129, 129, True, {"y": TC, "z1": TC, "z2": F32}),
    "dag_tc_then_fp32": (lambda a: _stemmed((8, 8), 32, a, [
        _conv("y", "x", 3, 1, 32, "same", a), _conv("z1", "y", 1, 2, 16, "valid", a), _conv("z2", "y", 3, 1, 32, "same", a)],
        ["z1", "z2"]), 64, 64, False, {"y": TC, "z1": F32, "z2": TC}),
    "dag_two_dense": (lambda a: _stemmed((4, 4), 32, a, [
        _conv("y", "x", 3, 1, 32, "same", a), _dense("z1", "y", 16, a), _dense("z2", "y", 64, a), _dense("z3", "z2", 32, a)],
        ["z1", "z3"]), 200, 200, False, {"y": TC, "z1": dict(tc=True, n_dg=64), "z2": TC, "z3": dict(tc=True, n_dg=64)}),
    # fallbacks to the fp32 kernels and the hand-offs tc -> fp32 -> tc
    "fb_cin8": (lambda a: _stemmed((6, 6), 8, a, [_conv("y", "x", 3, 1, 16, "same", a), _conv("z", "y", 3, 1, 32, "same", a)],
                                   ["z"]), 65, 65, False, {"x": F32, "y": F32, "z": TC}),
    "fb_cout80": (lambda a: _stemmed((6, 6), 16, a, [_conv("y", "x", 3, 1, 80, "same", a), _dense("z", "y", 16, a)], ["z"]),
                  63, 63, True, {"x": TC, "y": F32, "z": TC}),
    "fb_stride_over_k": (lambda a: _stemmed((8, 8), 32, a, [_conv("y", "x", 1, 2, 32, "valid", a),
                                                            _conv("z", "y", 3, 1, 16, "same", a)], ["z"]),
                         129, 129, False, {"x": TC, "y": F32, "z": TC}),
    "fb_r_over_32": (_one_conv((8, 8), 64, 16, 9, 1, "same"), 64, 64, False, {"x": TC, "y": F32}),
    "fb_dense_k40": (lambda a: _stemmed((2, 2), 16, a, [_dense("y", "x", 40, a), _dense("z", "y", 16, a), _dense("w", "z", 32, a)],
                                        ["w"]), 65, 65, True, {"x": TC, "y": F32, "z": F32, "w": TC}),
    # dense layers: partial M tiles of the weight gradient, N = 48 as 16-wide tiles, split-K on and off
    "dense_48x16": (_dense_pair(48, 16), 1, 1, False, {"x": F32, "y": dict(tc=True, n_fwd=16, n_dg=16, k_slices=1)}),
    "dense_80x48": (_dense_pair(80, 48), 65, 65, True, {"y": dict(tc=True, n_fwd=16, n_dg=16, k_slices=1)}),
    "dense_144x96": (_dense_pair(144, 96), 129, 129, False, {"y": dict(tc=True, n_fwd=32, n_dg=16, k_slices=1)}),
    "dense_48x256": (_dense_pair(48, 256), 65, 65, False, {"y": dict(tc=True, n_fwd=64, n_dg=16)}),
    "dense_64x32_fused_bias": (lambda a: dict(input_dtype="float32", state_dim=(20,), scale=1.0, layers=[
        _dense("x", "obs", 64, a), _dense("y", "x", 64, a), _dense("z", "y", 32, a)], outputs=["z"]),
        65, 65, False, {"y": dict(tc=True, n_dg=64), "z": dict(tc=True, n_dg=64)}),
    "dense_4096x16": (_dense_4096(16), 129, 129, False, {"y": dict(tc=True, n_fwd=16, n_dg=64, k_slices=64)}),
    "dense_4096x96": (_dense_4096(96), 1, 1, True, {"y": dict(tc=True, n_fwd=32, n_dg=64, k_slices=32)}),
}


# ------------------------------------------------------------------------------------------- reference and runner
def _weights(arch, seed=11):
    w = orc.init_weights(arch, seed=seed)
    rng = np.random.default_rng(seed + 1)
    for k in w:                                   # non-zero biases so the bias paths are exercised
        if k.endswith("/bias"):
            w[k] = (rng.standard_normal(w[k].shape) * 0.05).astype(np.float32)
    return w


def _inputs(arch, B, gather, seed=2):
    rng = np.random.default_rng(seed)
    rows = B + 3 if gather else B
    shape = (rows,) + tuple(arch["state_dim"])
    if arch["input_dtype"] == "uint8":
        obs = rng.integers(0, 256, shape, dtype=np.uint8)
    else:
        obs = rng.standard_normal(shape).astype(np.float32)
    idx = rng.permutation(rows)[:B].astype(np.int32) if gather else None
    sizes = orc.tensor_shapes(arch)
    gh = {h: rng.standard_normal((B, int(np.prod(sizes[h])))).astype(np.float32) for h in arch["outputs"]}
    return obs, idx, gh


def _reference(arch, w, obs, prec, gh=None, masks=None):
    """Pre-activations of every layer in torch-CPU `prec`, and (gh given) the parameter gradients of
    sum_h pre_h . G_h.  A ReLU layer computes pre * masks[name] when masks are given, else relu(pre)."""
    dt = torch.float64 if prec == "f64" else torch.float32
    params = {k: torch.from_numpy(v).to(dt).requires_grad_(gh is not None) for k, v in w.items()}
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
        act = sp.get("act")
        if act == "relu":
            t[name] = p * torch.from_numpy(masks[name]).to(dt).reshape(p.shape) if masks is not None else torch.relu(p)
        else:
            t[name] = torch.tanh(p) if act == "tanh" else p
    pre_np = {n: v.detach().reshape(B, -1).numpy() for n, v in pre.items()}
    if gh is None:
        return pre_np, None
    loss = sum((pre[h].reshape(B, -1) * torch.from_numpy(gh[h]).to(dt)).sum() for h in arch["outputs"])
    loss.backward()
    return pre_np, {k: params[k].grad.numpy() for k in w}


def _gpu_run(net, arch, obs, idx, B, gh):
    """forward and backward on the device: every tensor [B, size] and the parameter gradients"""
    obs_d = dev(obs)
    idx_d = dev(idx) if idx is not None else None
    net.forward(obs_d, B, idx=idx_d)
    tens = {n: net.tensor(n)[:B].cpu().numpy() for n, _, _, _ in arch["layers"]}
    for h in arch["outputs"]:
        net.tensor_grad(h)[:B].copy_(dev(gh[h]))
    net.backward(obs_d, B, arch["outputs"], idx=idx_d)
    return tens, net.get_weights(net.grads)


def _check_parity(tag, arch, w, obs, idx, gh, gpu_t, gpu_g, tc):
    """float64 distances of one GPU run; asserts the bounds of the path (tc: tensor cores where planned)"""
    x = obs[idx] if idx is not None else obs
    with orc.precision("f64"):
        f64_t = {n: v.detach().reshape(x.shape[0], -1).numpy() for n, v in orc.forward(arch, w, x, keep=True).items() if n != "obs"}
    relu = [n for n, _, _, sp in arch["layers"] if sp.get("act") == "relu"]
    masks = None
    if relu:
        pre64, _ = _reference(arch, w, x, "f64")
        masks = {}
        for n in relu:
            m = gpu_t[n] > 0
            flip = m != (pre64[n] > 0)
            worst = float(np.abs(pre64[n][flip]).max()) if flip.any() else 0.0
            assert worst < MASK_TIE * float(np.abs(pre64[n]).max()), (n, int(flip.sum()), worst)
            masks[n] = m
    _, f64_g = _reference(arch, w, x, "f64", gh, masks)
    fwd = {n: rel_err(gpu_t[n], f64_t[n]) for n in gpu_t}
    grd = {k: (l2_rel(gpu_g[k], f64_g[k]), rel_err(gpu_g[k], f64_g[k])) for k in w}
    if tc:
        bad = {n: e for n, e in fwd.items() if not e < TC_FWD_BOUND}
        bad.update({k: e for k, e in grd.items() if not (e[0] < TC_GRAD_BOUND and e[1] < REL)})
        rec = {"forward_max_rel": {n: "%.2e" % e for n, e in fwd.items()},
               "grad_l2_rel,max_rel": {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in grd.items()}}
    else:
        with orc.precision("f32"):
            f32_t = {n: v.detach().reshape(x.shape[0], -1).numpy() for n, v in orc.forward(arch, w, x, keep=True).items() if n != "obs"}
        _, f32_g = _reference(arch, w, x, "f32", gh, masks)
        cpu_f = {n: rel_err(f32_t[n], f64_t[n]) for n in fwd}
        cpu_g = {k: l2_rel(f32_g[k], f64_g[k]) for k in w}
        bad = {n: (e, cpu_f[n]) for n, e in fwd.items() if not e <= 2 * cpu_f[n] + F32_FLOOR}
        bad.update({k: (e[0], cpu_g[k]) for k, e in grd.items() if not e[0] <= 2 * cpu_g[k] + F32_FLOOR})
        rec = {"forward_max_rel(gpu,cpu32)": {n: ["%.2e" % e, "%.2e" % cpu_f[n]] for n, e in fwd.items()},
               "grad_l2_rel(gpu,cpu32)": {k: ["%.2e" % e[0], "%.2e" % cpu_g[k]] for k, e in grd.items()}}
    _record(tag, rec)
    assert not bad, bad


def _plan(net, arch):
    return {name: net.layer_plan(i) for i, (name, _, _, _) in enumerate(arch["layers"])}


def _assert_plan(plan, expect):
    for name, fields in expect.items():
        got = {k: plan[name][k] for k in fields}
        assert got == fields, (name, got, fields)


# ------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("act", ["tanh", "relu"])
@pytest.mark.parametrize("case", list(CASES))
def test_layer_sweep(xb, tc_mode, case, act):
    from xingtian_b200.engine import Net
    make, B, max_batch, gather, expect = CASES[case]
    arch = make(act)
    net = Net(arch, max_batch=max_batch)
    _assert_plan(_plan(net, arch), expect)
    w = _weights(arch)
    net.set_weights(w)
    obs, idx, gh = _inputs(arch, B, gather)
    gpu_t, gpu_g = _gpu_run(net, arch, obs, idx, B, gh)
    _check_parity("layer_sweep/%s/%s/B%d/%s" % (case, act, B, "tcgen05" if tc_mode else "fp32"),
                  arch, w, obs, idx, gh, gpu_t, gpu_g, tc_mode)


def _accumulates(arch, plan):
    """tensors whose gradient two tensor-core layers write (the second one through the `accumulate` epilogue)"""
    readers = {}
    for name, _, src, _ in arch["layers"]:
        if plan[name]["tc"]:
            readers[src] = readers.get(src, 0) + 1
    return [t for t, c in readers.items() if c >= 2 and t != "obs"]


def test_sweep_covers_the_tensor_core_plan(xb):
    """The union of the sweep's tensor-core layers reaches every kernel form it was written for."""
    from xingtian_b200.engine import Net
    seen = set()
    for case, (make, B, max_batch, gather, expect) in CASES.items():
        arch = make("tanh")
        net = Net(arch, max_batch=max_batch)
        plan = _plan(net, arch)
        for name, kind, src, sp in arch["layers"]:
            p = plan[name]
            if not p["tc"]:
                continue
            if p["kind"] == "conv":
                seen.add(("conv fwd", p["n_fwd"]))
                seen.add(("conv wgrad", sp["cout"]))
                if src != "obs":
                    seen.add(("conv dgrad", p["n_dg"]))
                seen.add(("w_res", p["w_res"]))
                if p["dg_empty_units"] and src != "obs":
                    seen.add("empty unit")
                if p["s2d"]:
                    seen.add("s2d")
            else:
                seen.add(("dense split-K", p["k_slices"] > 1))
        if _accumulates(arch, plan):
            seen.add("accumulate")
        del net
    want = {(form, n) for form in ("conv fwd", "conv dgrad", "conv wgrad") for n in (16, 32, 48, 64)}
    want |= {("w_res", True), ("w_res", False), "empty unit", "accumulate", "s2d", ("dense split-K", True), ("dense split-K", False)}
    assert not want - seen, sorted(map(str, want - seen))


def _reuse_arch(act="tanh"):
    # empty data-gradient units (y) and a tensor read by two tensor-core convs (x: accumulate)
    return _stemmed((10, 10), 32, act, [_conv("y", "x", 3, 2, 48, "valid", act), _conv("z", "x", 3, 1, 32, "same", act)], ["y", "z"])


def test_net_reused_at_smaller_batch(xb, tc_mode):
    """Gradient-plane rows in [B, round16(B)) are read by the weight-gradient K loop: after a B = 200 pass, a B = 37 pass
    on the same net must give what a fresh net gives at B = 37."""
    from xingtian_b200.engine import Net
    arch = _reuse_arch()
    w = _weights(arch)
    used = Net(arch, max_batch=200)
    used.set_weights(w)
    plan = _plan(used, arch)
    assert plan["y"]["dg_empty_units"] > 0 and _accumulates(arch, plan) == ["x"]
    obs, idx, gh = _inputs(arch, 200, True, seed=5)
    _gpu_run(used, arch, obs, idx, 200, gh)
    obs, idx, gh = _inputs(arch, 37, True, seed=6)
    got = _gpu_run(used, arch, obs, idx, 37, gh)
    fresh = Net(arch, max_batch=200)
    fresh.set_weights(w)
    ref1 = _gpu_run(fresh, arch, obs, idx, 37, gh)
    ref2 = _gpu_run(fresh, arch, obs, idx, 37, gh)

    def same(a, b):
        return all(np.array_equal(a[i][k], b[i][k]) for i in range(2) for k in a[i])
    if same(ref1, ref2):
        for i in range(2):
            for k in got[i]:
                np.testing.assert_array_equal(got[i][k], ref1[i][k], err_msg=k)
    else:       # the fresh net is not bitwise reproducible: hold the reused one to the float64 bounds
        _check_parity("net_reuse/B37/%s" % ("tcgen05" if tc_mode else "fp32"), arch, w, obs, idx, gh, got[0], got[1], tc_mode)


@pytest.mark.parametrize("hw,on_tc", [((42, 42), False), ((24, 24), True)])
def test_large_map_conv_falls_back(xb, tc_mode, hw, on_tc):
    """A 3x3 SAME 32 -> 32 conv on a 42 x 42 map has a data-gradient stage table (127 KB) that leaves its launch one ring
    stage, and a weight-gradient table that does not fit beside the four weight-gradient stages: it must be planned off
    the tensor cores (or onto launches that fit) and still compute forward and backward.  24 x 24 stays on them."""
    from xingtian_b200.engine import Net
    arch = _one_conv(hw, 32, 32, 3, 1, "same")("tanh")
    B = 9
    net = Net(arch, max_batch=B)
    p = net.layer_plan(1)
    assert p["tc"] == on_tc, p
    if p["tc"]:
        assert p["fwd_stages"] >= 2 and p["dg_stages"] >= 2, p
    assert net.layer_plan(0)["tc"]
    w = _weights(arch)
    net.set_weights(w)
    obs, idx, gh = _inputs(arch, B, False)
    gpu_t, gpu_g = _gpu_run(net, arch, obs, idx, B, gh)
    _check_parity("large_map/%dx%d/%s" % (hw + ("tcgen05" if tc_mode else "fp32",)), arch, w, obs, idx, gh, gpu_t, gpu_g, tc_mode)
