"""Categorical PPO's fused heads against float64 in every instantiation they have, on both kernel paths, with fused
heads on and off:

- the train step (heads_kernel<PpoLoss, kpl, amax>): PpoMlp [4] -> A at LR 0, so every minibatch of a call sees the
  same weights and each entry of the loss trace, and the last minibatch's gradient bucket, compare with float64
  directly.  Cases reach every entry of the train table, the grid-stride regime (more than 132 blocks x 8 warps = 1056
  samples: a warp sums several samples' weight gradients), a ragged minibatch after full ones (plane rows [mb,
  round16(mb)) must be re-zeroed), the layer path at its edges (K % 32, A up to MAX_ADIM = 32, K beyond 512) and
  PpoCnn at the benchmark's shape;
- rollout inference (infer_heads_kernel<Categorical, kpl, amax>, or the forward and sample_kernel): actions, log-probs,
  values and the last step's logits against float64 with the Philox uniforms of each (env, step), one and many steps
  per chunk, ragged last chunks, grid-stride chunks and every entry of the inference table.

Every case asserts the instantiation it is named for (xtb_ppo_heads_plan), and test_cases_cover_every_heads_instantiation
that together they reach every entry the library can launch."""
import collections

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from test_gpu_activations import _restore_module_config  # noqa: F401
from test_gpu_kernels import RELU_FLIP_F32, RELU_FLIP_TC, _keepalive, l2_rel, rel_err, tc_mode, xb  # noqa: F401
from test_gpu_ppo_gauss import _desc, _eager_launches

pytestmark = pytest.mark.gpu

LAYERS = (0, 0)      # the plan of heads that run layer by layer
HEADS = ("pi_latent/kernel", "pi_latent/bias", "output_value/kernel", "output_value/bias")
# The heads of PpoCnn on the tensor-core path, fused or not: the bf16x3 conv trunk moves the values by 1.3e-6 on average,
# all the same way, and the value head's gradients are sums over 4096 samples that cancel (the bias gradient to 1.2e-3),
# so they carry it: observed 5.0e-4 (output_value/bias) and 2.0e-4 (output_value/kernel) on an H100, where the float64
# gradient taken from the device's own values agrees with the device's to 2e-7
CNN_TC_HEADS = 1e-3


class Case(collections.namedtuple("Case", "K A B plan shared act cnn ragged depth")):
    """K hidden units in each of `depth` hidden layers, A actions, B samples in one minibatch (ragged: N = 2 B + 45
    samples in minibatches of B); plan: the (kpl, amax) of the heads_kernel entry the fused call launches, LAYERS when
    it runs layer by layer"""

    @property
    def id(self):
        reg = "layers" if self.plan == LAYERS else "fused%dx%d" % self.plan
        s = "%s-K%d-A%d-%s%d" % (reg, self.K, self.A, "N" if self.ragged else "B", self.n if self.ragged else self.B)
        tags = (("shared", self.shared), (self.act, self.act != "tanh"), ("cnn", self.cnn), ("ragged", self.ragged),
                ("%dlayers" % self.depth, self.depth != 2 and not self.cnn))
        return s + "".join("-" + t for t, on in tags if on)

    @property
    def n(self):
        return 2 * self.B + 45 if self.ragged else self.B


def _case(K, A, B, plan, shared=False, act="tanh", cnn=False, ragged=False, depth=2):
    return Case(K, A, B, plan, shared, act, cnn, ragged, 1 if cnn else depth)


TRAIN = [
    # (2, 8): K <= 64, A <= 8 -- A = 1: logp is 0 and the entropy 0
    _case(32, 2, 37, (2, 8)), _case(64, 8, 17, (2, 8)), _case(64, 1, 37, (2, 8)), _case(64, 2, 37, (2, 8), shared=True),
    # (8, 4): B = 1057 gives the first warp a second sample, 4096 is C5's minibatch
    _case(96, 3, 37, (8, 4)), _case(256, 4, 1, (8, 4)), _case(256, 4, 1057, (8, 4)), _case(256, 4, 4096, (8, 4)),
    _case(96, 5, 37, (8, 8)), _case(256, 8, 200, (8, 8)),
    # (16, 4): hidden units 256..511
    _case(288, 2, 37, (16, 4)), _case(512, 4, 17, (16, 4)), _case(512, 4, 4096, (16, 4)),
    # layer by layer even when fused: K % 32, A > 8, A = MAX_ADIM (8 Philox groups), K = 288 with A = 5, K > 512, and
    # K = 512 with A = 8, which infers fused but trains layer by layer
    _case(48, 4, 37, LAYERS), _case(64, 9, 37, LAYERS), _case(64, 32, 200, LAYERS), _case(288, 5, 37, LAYERS),
    _case(544, 2, 37, LAYERS), _case(512, 8, 37, LAYERS),
    # a 45-sample minibatch after two of 320: the planes of its rows [45, 48) held the previous minibatch's gradients.
    # The weight gradient of the heads' hidden layer multiplies those rows with the same rows of its input, which are
    # zero when that input was converted from fp32 (the first hidden layer reads the observation and runs in fp32),
    # but hold the previous minibatch's values when a tensor-core layer wrote it: hence three hidden layers
    _case(256, 4, 320, (8, 4), shared=True, ragged=True), _case(512, 4, 320, (16, 4), ragged=True),
    _case(256, 4, 320, (8, 4), ragged=True, depth=3),
    _case(256, 4, 320, (8, 4), shared=True, act="relu"),
    # the benchmark's PpoCnn: 84x84x4 uint8 frames, relu [256], one tower, one minibatch of 4096
    _case(256, 4, 4096, (8, 4), shared=True, act="relu", cnn=True),
]


class RolloutCase(collections.namedtuple("RolloutCase", "K A E T M plan cnn")):
    """E environments, T steps, max_predict_batch M (M // E steps per chunk); plan: the infer_heads_kernel entry.
    PpoMlp with tanh separate towers [K, K], or PpoCnn with relu and one tower [K]"""
    shared = property(lambda self: self.cnn)
    act = property(lambda self: "relu" if self.cnn else "tanh")
    depth = property(lambda self: 1 if self.cnn else 2)

    @property
    def id(self):
        reg = "layers" if self.plan == LAYERS else "fused%dx%d" % self.plan
        return "%s-K%d-A%d-E%d-T%d-M%d%s" % (reg, self.K, self.A, self.E, self.T, self.M, "-cnn" if self.cnn else "")


def _rcase(K, A, E, T, M, plan, cnn=False):
    return RolloutCase(K, A, E, T, M, plan, cnn)


ROLLOUT = [
    # one step per chunk
    _rcase(64, 8, 37, 3, 64, (2, 8)), _rcase(256, 4, 37, 3, 64, (8, 4)), _rcase(96, 5, 37, 3, 64, (8, 8)),
    _rcase(512, 8, 37, 3, 64, (16, 8)), _rcase(288, 5, 37, 3, 64, (16, 8)),
    # many steps per chunk: 320, 320 and 60 steps of one env; chunks of 2, 2 and 1 steps
    _rcase(256, 4, 1, 700, 320, (8, 4)), _rcase(256, 8, 150, 5, 320, (8, 8)),
    # grid-stride: C5's chunk of 8 steps x 512 envs, and 2 x 1057 rows
    _rcase(256, 4, 512, 8, 4096, (8, 4)), _rcase(512, 4, 1057, 2, 4096, (16, 8)),
    # layer by layer: K % 32, A = MAX_ADIM (8 Philox groups), A > 8
    _rcase(48, 4, 37, 3, 64, LAYERS), _rcase(64, 32, 37, 3, 64, LAYERS), _rcase(64, 9, 37, 3, 64, LAYERS),
    # the benchmark's C5 inference: PpoCnn relu [256], 8 steps x 512 envs in one chunk
    _rcase(256, 4, 512, 8, 4096, (8, 4), cnn=True),
]


def _model(c, batch, max_predict=1024):
    """Categorical PpoMlp [4] -> A with `depth` hidden layers of K (or PpoCnn 84x84x4 uint8 with [K]) at LR 0, one
    epoch, graphs off (the launches are counted), with non-zero biases: at their initial zeros every layer maps a zero
    row to zero, which hides a kernel that reads rows past the batch"""
    import xingtian_b200  # noqa: F401
    from xingtian_b200.registry import Registers
    cfg = {"BATCH_SIZE": batch, "NUM_SGD_ITER": 1, "LR": 0.0, "hidden_sizes": [c.K] * c.depth, "activation": c.act,
           "VF_SHARE_LAYERS": c.shared, "action_type": "Categorical", "init_seed": 3, "VF_CLIP": 0.5, "ENTROPY_LOSS": 0.01,
           "LOSS_CLIPPING": 0.2, "use_cuda_graph": False}
    info = {"state_dim": [84, 84, 4] if c.cnn else [4], "action_dim": c.A, "input_dtype": "uint8" if c.cnn else "float32",
            "max_predict_batch": max_predict, "model_config": cfg}
    m = Registers.model["PpoCnn" if c.cnn else "PpoMlp"](info)
    rng = np.random.default_rng(c.K * 64 + c.A)
    m.set_weights({k: (v + 0.1 * rng.standard_normal(v.shape)).astype(np.float32) if k.endswith("/bias") else v
                   for k, v in m.get_weights().items()})
    return m


def _arch(c):
    if c.cnn:
        return orc.ppo_cnn_arch(action_dim=c.A, hidden_sizes=(c.K,), activation=c.act, vf_share_layers=c.shared)
    return orc.ppo_mlp_arch(state_dim=(4,), action_dim=c.A, hidden_sizes=(c.K,) * c.depth, activation=c.act,
                            vf_share_layers=c.shared)


def _obs(c, rows, rng):
    if c.cnn:
        return rng.integers(0, 256, (rows, 84, 84, 4), dtype=np.uint8)
    return rng.standard_normal((rows, 4)).astype(np.float32)


# ---- the train step -------------------------------------------------------------------------------------------------
def _step_data(c, arch, w, seed):
    """N samples whose ratios reach both sides of the surrogate clip and whose values pass the value clip"""
    rng = np.random.default_rng(seed)
    obs = _obs(c, c.n, rng)
    with torch.no_grad():
        logits, v = orc.forward(arch, w, obs)
    act = rng.integers(0, c.A, c.n).astype(np.int32)
    with orc.precision("f64"):
        lp = orc.categorical_logp(logits.double(), torch.from_numpy(act)).numpy()
    old_logp = (lp + 0.5 * rng.standard_normal((c.n, 1))).astype(np.float32)
    old_v = (v.numpy() + 1.5 * rng.standard_normal((c.n, 1))).astype(np.float32)
    label = [act, old_logp, rng.standard_normal((c.n, 1)).astype(np.float32), old_v,
             rng.standard_normal((c.n, 1)).astype(np.float32)]
    return obs, label, np.exp(lp - old_logp), np.abs(v.numpy() - old_v)


def _oracle_mb(arch, w, obs, label, idx, dt, grads):
    with orc.precision(dt):
        ref = orc.PpoLearner(arch, w, batch_size=len(idx), ent_coef=0.01, clip_ratio=0.2, num_sgd_iter=1, vf_clip=0.5)
        loss, g = ref.loss_and_grads(obs[idx], *[x[idx] for x in label])
        return float(loss), ({k: t.detach().numpy() for k, t in zip(ref.names, g)} if grads else None)


_TRAIN_REF = {}     # case id -> data, minibatches and the float64 / fp32 oracle (independent of kernel path and fuse)


def _train_reference(c, m):
    if c.id not in _TRAIN_REF:
        arch, w = _arch(c), m.get_weights()
        assert list(w) == list(orc.param_shapes(arch))
        obs, label, ratio, vdev = _step_data(c, arch, w, seed=c.K * 7 + c.A * 100 + c.B)
        np.random.seed(0)
        perm = m.make_perm(c.n)
        mbs = [perm[0, s:s + c.B] for s in range(0, c.n, c.B)]
        refs = []
        for j, idx in enumerate(mbs):
            last = j == len(mbs) - 1
            refs.append((_oracle_mb(arch, w, obs, label, idx, "f64", last), _oracle_mb(arch, w, obs, label, idx, "f32", last)))
        _TRAIN_REF[c.id] = dict(w=w, obs=obs, label=label, ratio=ratio, vdev=vdev, perm=perm, refs=refs)
    return _TRAIN_REF[c.id]


@pytest.mark.parametrize("c", TRAIN, ids=[c.id for c in TRAIN])
def test_train_step_against_float64(xb, tc_mode, c):
    """fused heads on and off: the plan each launches, fewer launches fused (the same number where both run layer by
    layer), weights untouched at LR 0, every loss of the call and the last minibatch's gradients at most 4x torch-CPU
    fp32's distance from float64 (+ the bf16x3 floor on the tensor-core path; ReLU trunks + the suite's flip
    allowance, PpoCnn's heads on the tensor cores + CNN_TC_HEADS)"""
    lib = xb["lib"]
    out = {}
    try:
        for fuse in (1, 0):
            lib.xtb_set_fuse_heads(fuse)
            m = _model(c, c.B)
            assert m.heads_plan(False) == (c.plan if fuse else LAYERS)
            ref = _train_reference(c, m)
            w0 = m.get_weights()
            for k in w0:
                assert np.array_equal(w0[k], ref["w"][k]), k
            m.upload_rollout([ref["obs"]], ref["label"])
            n = _eager_launches(lib, lambda: m.train_device(c.n, ref["perm"]))
            w1 = m.get_weights()
            for k in w0:
                assert np.array_equal(w1[k], w0[k]), k       # LR 0: every minibatch saw the initial weights
            out[fuse] = (n, np.array(m.last_losses, np.float64), m.net.get_weights(m.net.grads))
    finally:
        lib.xtb_set_fuse_heads(1)
    assert (out[1][0] < out[0][0]) if c.plan != LAYERS else (out[1][0] == out[0][0]), (out[1][0], out[0][0])
    if c.B >= 37:
        assert (ref["ratio"] < 0.8).any() and (ref["ratio"] > 1.2).any() and (ref["vdev"] > 0.5).any()
    # the bias gradients of the hidden layers are sums over B samples whose terms partly cancel: their relative
    # rounding error grows like sqrt(B) (as in test_gpu_ppo_gauss)
    floor = (6e-5 if tc_mode == 1 else 1e-5) * max(1.0, np.sqrt(c.B / 128.0))
    flip = (RELU_FLIP_TC if tc_mode == 1 else RELU_FLIP_F32) if c.act == "relu" else 0.0
    heads = CNN_TC_HEADS if (c.cnn and tc_mode == 1) else 0.0
    refs = ref["refs"]
    for fuse, (_, losses, g) in out.items():
        assert len(losses) == len(refs)
        for j, ((l64, _), (l32, _)) in enumerate(refs):
            assert abs(losses[j] - l64) <= 4 * abs(l32 - l64) + floor * max(1.0, abs(l64)), (fuse, j, losses[j], l64, l32)
        (_, g64), (_, g32) = refs[-1]
        bad = {k: (l2_rel(g[k], g64[k]), l2_rel(g32[k], g64[k])) for k in g64
               if not l2_rel(g[k], g64[k]) <= 4 * l2_rel(g32[k], g64[k]) + floor + (heads if k in HEADS else flip)}
        assert not bad, (fuse, bad)


# ---- rollout inference ----------------------------------------------------------------------------------------------
_ROLLOUT_REF = {}   # case id -> weights, observations and the float64 logits / values of every step


def _rollout_reference(c, m):
    if c.id not in _ROLLOUT_REF:
        arch, w = _arch(c), m.get_weights()
        obs = _obs(c, c.E * c.T, np.random.default_rng(c.K + c.A * 10 + c.E))
        w64 = {k: v.astype(np.float64) for k, v in w.items()}
        logits, values = [], []
        with orc.precision("f64"), torch.no_grad():
            for t in range(c.T):
                lg, v = orc.forward(arch, w64, obs[t * c.E:(t + 1) * c.E])
                logits.append(lg.numpy()); values.append(v.numpy().ravel())
        _ROLLOUT_REF[c.id] = dict(w=w, obs=obs, logits=np.stack(logits), values=np.stack(values))
    return _ROLLOUT_REF[c.id]


@pytest.mark.parametrize("c", ROLLOUT, ids=[c.id for c in ROLLOUT])
def test_rollout_infer_against_float64(xb, tc_mode, c):
    """rollout inference with fused heads on and off: the plan, fewer launches fused (the same number layer by layer),
    the draw of every (env, step) against float64 Gumbel-argmax on the Philox uniforms, log-probs and values, the last
    step's logits in rows [0, E) of the pi head and the offset counter advanced by T"""
    lib = xb["lib"]
    E, T, A = c.E, c.T, c.A
    res = {}
    try:
        for fuse in (1, 0):
            lib.xtb_set_fuse_heads(fuse)
            m = _model(c, c.M, max_predict=c.M)
            assert m.net.max_batch == c.M
            assert m.heads_plan(True) == (c.plan if fuse else LAYERS)
            ref = _rollout_reference(c, m)
            w = m.get_weights()
            for k in w:
                assert np.array_equal(w[k], ref["w"][k]), k
            obs_d = torch.from_numpy(ref["obs"]).cuda()
            act = torch.empty(T, E, dtype=torch.int32, device="cuda")
            lp = torch.empty(T, E, device="cuda"); val = torch.empty(T, E, device="cuda")
            m._offset_dev = torch.zeros(1, dtype=torch.int64, device="cuda")
            n = _eager_launches(lib, lambda: m.rollout_infer_device(obs_d, None, E, T, act, lp, val))
            res[fuse] = (n, act.cpu().numpy(), lp.cpu().numpy(), val.cpu().numpy(),
                         m.net.tensor("pi_latent")[:E].cpu().numpy(), int(m._offset_dev.cpu()[0]), m._sample_seed)
    finally:
        lib.xtb_set_fuse_heads(1)
    assert (res[1][0] < res[0][0]) if c.plan != LAYERS else (res[1][0] == res[0][0]), (res[1][0], res[0][0])
    lg64, v64 = ref["logits"], ref["values"]
    for fuse, (_, a_g, l_g, v_g, head, off, seed) in res.items():
        assert off == T
        u = np.stack([orc.philox_uniforms(seed, t, E, A) for t in range(T)]).astype(np.float64)
        score = lg64 - np.log(-np.log(u))
        want = np.argmax(score, axis=-1)
        top2 = np.argsort(score, axis=-1)[..., -2:]
        srt = np.take_along_axis(score, top2, axis=-1)
        tie = srt[..., 1] - srt[..., 0] < 1e-4
        miss = a_g != want
        # expf / logf on the device differ from float64 by ulps: a different draw is legal only on a near-tie
        assert not (miss & ~(tie & (top2 == a_g[..., None]).any(-1))).any(), (fuse, np.argwhere(miss)[:5])
        assert miss.mean() < 0.01, (fuse, miss.mean())
        with orc.precision("f64"):
            lp64 = orc.categorical_logp(torch.from_numpy(lg64.reshape(T * E, A)), torch.from_numpy(a_g.reshape(-1))).numpy()
        assert rel_err(l_g.ravel(), lp64.ravel()) <= 1e-4, (fuse, rel_err(l_g.ravel(), lp64.ravel()))
        assert rel_err(v_g, v64) <= 1e-4, (fuse, rel_err(v_g, v64))
        assert rel_err(head, lg64[-1]) <= 1e-4, (fuse, rel_err(head, lg64[-1]))


# ---- the cases reach every instantiation ----------------------------------------------------------------------------
def _library_plans(xb, K_max=1024):
    """every (kpl, amax) the library launches for some dense heads (K hidden units, A actions) in training and in
    inference, from xtb_ppo_heads_plan on one-tower nets over the whole width and action range"""
    import ctypes as C
    capi, lib = xb["capi"], xb["lib"]
    plans = {False: set(), True: set()}
    lib.xtb_set_fuse_heads(1)
    for K in range(32, K_max + 1, 32):
        for A in range(1, 33):
            h = C.c_void_p()
            assert lib.xtb_net_create(C.byref(_desc(capi, [(capi.DENSE, 0, capi.ACT["tanh"], K), (capi.DENSE, 1, 0, A),
                                                            (capi.DENSE, 1, 0, 1)], in_dim=4)), 8, C.byref(h)) == 0
            try:
                for infer in (False, True):
                    kpl, amax = C.c_int(), C.c_int()
                    assert lib.xtb_ppo_heads_plan(h, 2, 3, int(infer), C.byref(kpl), C.byref(amax)) == 0
                    plans[infer].add((kpl.value, amax.value))
            finally:
                lib.xtb_net_destroy(h)
    return {k: v - {LAYERS} for k, v in plans.items()}


def test_cases_cover_every_heads_instantiation(xb):
    """the train cases reach every heads_kernel entry and the rollout cases every infer_heads_kernel entry the library
    can pick; a new table entry needs a case that reaches it"""
    import ctypes as C
    lib = xb["lib"]
    lib_plans = _library_plans(xb)
    assert lib_plans[False] and lib_plans[True]
    assert {c.plan for c in TRAIN} - {LAYERS} == lib_plans[False]
    assert {c.plan for c in ROLLOUT} - {LAYERS} == lib_plans[True]
    assert {c.plan for c in TRAIN} >= {LAYERS} and {c.plan for c in ROLLOUT} >= {LAYERS}
    # the heads-plan query checks its arguments like the other PPO calls, without a launch
    h = C.c_void_p()
    capi = xb["capi"]
    assert lib.xtb_net_create(C.byref(_desc(capi, [(capi.DENSE, 0, capi.ACT["tanh"], 64), (capi.DENSE, 1, 0, 3),
                                                    (capi.DENSE, 1, 0, 1)], in_dim=4)), 8, C.byref(h)) == 0
    try:
        before = lib.xtb_launch_count()
        kpl, amax = C.c_int(7), C.c_int(7)
        for pi_t, v_t in ((0, 3), (2, 4), (3, 2), (2, 2)):      # out of range, or a value head wider than 1
            assert lib.xtb_ppo_heads_plan(h, pi_t, v_t, 0, C.byref(kpl), C.byref(amax)) == -1
        assert lib.xtb_ppo_heads_plan(None, 2, 3, 0, C.byref(kpl), C.byref(amax)) == -1
        assert lib.xtb_ppo_heads_plan(h, 2, 3, 0, None, C.byref(amax)) == -1
        assert lib.xtb_launch_count() == before and (kpl.value, amax.value) == (7, 7)
        try:
            lib.xtb_set_fuse_heads(0)
            assert lib.xtb_ppo_heads_plan(h, 2, 3, 1, C.byref(kpl), C.byref(amax)) == 0 and (kpl.value, amax.value) == LAYERS
        finally:
            lib.xtb_set_fuse_heads(1)
    finally:
        lib.xtb_net_destroy(h)
