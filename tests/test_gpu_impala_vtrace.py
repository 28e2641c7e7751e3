"""IMPALA's V-trace learner step (ImpalaCnnOpt through xtb_impala_train) against float64:

a. vtrace_kernel through xtb_vtrace_loss_grad: vs, pg_adv, the logit and baseline gradients and the loss against the
   oracle's float64 V-trace and autograd, at the trajectory lengths where the warp's lane chunks change (T = S - 1 kept
   steps in chunks of (T + 31) / 32), trajectory counts that fill the last 128-thread block partly and exactly, one to
   MAX_ADIM = 32 actions, gamma 0 and 1, and the data regimes rho = 1, rho on both sides of 1 and rho overflowing fp32;
   plus its contract: every output written, row S - 1 zero and without effect, vs / pg optional, loss accumulated, bad
   arguments refused without a launch;
b. the learner step at LR 0: loss, every parameter gradient and the global norm the optimiser saw, against float64 on
   both kernel paths (the product ImpalaCnnOpt with ReLU, and a tanh net called through the C-ABI);
c. the step's forms: eager, graph capture, graph replay and the data-parallel path with a one-rank communicator give
   the same loss, bitwise the same gradients for the layers on the tensor cores, and the others up to the order of
   atomic fp32 sums;
d. the clip and Adam wiring of one step at LR 5e-4 whose gradient norm exceeds the clip.

Every observed error is recorded through tests/parity_record.py."""
import collections

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
from parity_record import record
from test_gpu_kernels import RELU_FLIP_F32, RELU_FLIP_TC, _keepalive, dev, l2_rel, one_rank_comm, rel_err, tc_mode, xb  # noqa: F401

pytestmark = pytest.mark.gpu

XTB_ERR_ARG = -1
MAX_ADIM = 32
# a few fp32 ulps on top of 4 x the fp32 oracle's distance from float64 (observed on an H100 80GB HBM3 at 700 W: at most
# 26 % of the bound, the largest errors 3.3e-5 on dlogits with extreme logits, where the fp32 oracle has 3.3e-5 too)
VT_FLOOR = 2e-6


def _f32(x):
    """the value a C float argument carries"""
    return float(np.float32(x))


@pytest.fixture(scope="module", autouse=True)
def _restore_impala_config():
    """import_config writes each model config into xingtian_b200.model.impala's globals: restore them after the module"""
    from xingtian_b200.model import impala
    saved = {k: getattr(impala, k) for k in ("LR", "GAMMA", "ENTROPY_LOSS")}
    yield
    for k, v in saved.items():
        setattr(impala, k, v)


# ---- a. xtb_vtrace_loss_grad ----------------------------------------------------------------------------------------
class VCase(collections.namedtuple("VCase", "S k A gamma logits dones")):
    """k trajectories of S steps, A actions; logits: "equal" (behaviour = target, rho = 1), "near" (rho on both sides
    of 1) or "extreme" (|logits| up to 60, rho overflows fp32); dones: "random" (~5 %), "all", "lane_starts" (done at
    each lane's first step t0 = lane * chunk) or "last" (done at T - 1 only)"""

    @property
    def id(self):
        return "S%d-k%d-A%d-g%g-%s-%s" % (self.S, self.k, self.A, self.gamma, self.logits, self.dones)


VTRACE = [
    # the shapes of the fp32-oracle test this replaces: (k, S, A) = (4, 128, 4), (64, 128, 4), (1, 2, 4), (3, 50, 6)
    VCase(128, 4, 4, 0.99, "near", "random"), VCase(128, 64, 4, 0.99, "near", "random"),
    VCase(2, 1, 4, 0.99, "extreme", "last"), VCase(50, 3, 6, 0.99, "near", "random"),
    # T = 1 (above, S = 2): one lane.  T < 32: lanes idle; T = 2 and 31, one step per lane, the scan carries across lanes
    VCase(3, 5, 2, 0.99, "equal", "last"), VCase(32, 3, 1, 0.99, "equal", "last"),
    # T = 32: one step per lane; T = 33: 17 lanes, the last with one step
    VCase(33, 5, 32, 0.99, "near", "random"), VCase(34, 4, 18, 0.99, "extreme", "random"),
    VCase(33, 4, 2, 0.99, "near", "all"),
    # 257 trajectories: 65 blocks, the last with one warp; 64: 16 full blocks
    VCase(65, 257, 4, 0.99, "near", "random"), VCase(129, 64, 6, 0.99, "near", "last"),
    VCase(65, 5, 18, 0.99, "extreme", "last"), VCase(129, 1, 1, 0.99, "equal", "lane_starts"),
    # gamma = 0: no bootstrap at all
    VCase(50, 4, 4, 0.0, "near", "random"),
    # S = 1000: chunks of 32 steps; gamma = 1: the scan never decays (and without dones nothing cuts it)
    VCase(1000, 3, 4, 1.0, "near", "random"), VCase(1000, 5, 6, 1.0, "equal", "last"),
    VCase(1000, 1, 32, 0.99, "extreme", "lane_starts"),
]


def _vtrace_data(c):
    """env-major rows [k * S]; row S - 1 of each trajectory carries arbitrary values (only its baseline is read)"""
    rng = np.random.default_rng(c.S * 1000 + c.k * 10 + c.A)
    N, S, T, A = c.k * c.S, c.S, c.S - 1, c.A
    act = rng.integers(0, A, N).astype(np.int32)
    if c.logits == "extreme":
        assert A >= 2
        tp = rng.uniform(-60, 60, (N, A)).astype(np.float32)
        bp = rng.uniform(-60, 60, (N, A)).astype(np.float32)
        # every 5th row: log pi(a) >= -log A against log mu(a) <= -120: rho = e^116 and more, beyond fp32
        r = np.arange(0, N, 5)
        tp[r, act[r]] = 60.0
        bp[r] = 60.0
        bp[r, act[r]] = -60.0
    else:
        tp = (2 * rng.standard_normal((N, A))).astype(np.float32)
        bp = tp.copy() if c.logits == "equal" else (tp + 0.5 * rng.standard_normal((N, A))).astype(np.float32)
    base = (2 * rng.standard_normal(N)).astype(np.float32)
    rew = (2 * rng.standard_normal(N)).astype(np.float32)      # mostly beyond +-1: clipped
    rew[0::7], rew[3::7], rew[5::7] = 1.0, -1.0, 0.0
    done = np.zeros((c.k, S), bool)
    if c.dones == "random":
        done = rng.random((c.k, S)) < 0.05
    elif c.dones == "all":
        done[:] = True
    elif c.dones == "lane_starts":
        done[:, 0:T:(T + 31) // 32] = True
    else:
        done[:, T - 1] = True
    done[:, S - 1] = rng.random(c.k) < 0.5
    return dict(tp=tp, bp=bp, base=base, act=act, done=done.reshape(N), rew=rew)


def _kept(c):
    return np.arange(c.k * c.S) % c.S != c.S - 1


def _assert_regimes(c, d):
    """each regime the case is named for occurs on the rows the kernel reads"""
    kept = _kept(c)
    with np.errstate(over="ignore"):
        lp = lambda x, dt: (x.astype(dt) - x.astype(dt).max(-1, keepdims=True))  # noqa: E731
        lsm = lambda x, dt: lp(x, dt) - np.log(np.exp(lp(x, dt)).sum(-1, keepdims=True))  # noqa: E731
        pick = lambda x, dt: np.take_along_axis(lsm(x, dt), d["act"][:, None].astype(np.int64), 1)[:, 0]  # noqa: E731
        rho64 = np.exp(pick(d["tp"], np.float64) - pick(d["bp"], np.float64))[kept]
        rho32 = np.exp(pick(d["tp"], np.float32) - pick(d["bp"], np.float32))[kept]
    if c.logits == "equal":
        assert (rho64 == 1.0).all()
    elif c.logits == "near":
        assert (rho64 < 1).any() and (rho64 > 1).any()
    else:
        assert np.isinf(rho32).any() and np.abs(d["tp"]).max() > 59
    r = d["rew"][kept]
    if kept.sum() >= 7:
        assert (np.abs(r) > 1).any() and (r == 1).any() and (r == -1).any() and (r == 0).any()
    done = d["done"].reshape(c.k, c.S)[:, :c.S - 1]
    T = c.S - 1
    if c.dones == "random":
        assert done.any() and not done.all()
    elif c.dones == "all":
        assert done.all()
    elif c.dones == "lane_starts":
        chunk = (T + 31) // 32
        starts = np.arange(0, T, chunk)
        assert chunk >= 2 and done[:, starts].all() and done.sum() == c.k * len(starts)
    else:
        assert done[:, T - 1].all() and done.sum() == c.k
    # with more than one lane, the value a lane receives from the cross-lane scan reaches its last step: that step
    # carries a trace coefficient disc * min(1, rho) well above zero somewhere
    chunk = (T + 31) // 32
    if T > chunk and c.dones != "all" and c.gamma > 0:
        ends = np.arange(chunk, T, chunk) - 1
        coef = c.gamma * ~done[:, ends] * np.minimum(1.0, rho64.reshape(c.k, T)[:, ends])
        assert (coef > 0.1).any()


def _vtrace_reference(c, d, prec):
    """vs, pg_adv [k, S - 1], d loss / d logits [N, A], d loss / d baseline [N] and the loss, in `prec`"""
    f = np.float64 if prec == "f64" else np.float32
    g = _f32(c.gamma)
    with orc.precision(prec), np.errstate(over="ignore", under="ignore"):
        tpt = torch.from_numpy(d["tp"].astype(f)).requires_grad_(True)
        bt = torch.from_numpy(d["base"].astype(f)).requires_grad_(True)
        loss = orc.impala_loss(tpt, bt, d["bp"], d["act"], d["done"], d["rew"], c.S, gamma=g)
        loss.backward()
        sb = lambda x: orc.split_batches(x, c.S, True)  # noqa: E731
        vs, pg = orc.vtrace_from_logits(sb(d["bp"].astype(f)), sb(d["tp"].astype(f)), sb(d["act"]),
                                        sb((~d["done"]).astype(f) * f(g)), sb(np.clip(d["rew"].astype(f), -1, 1)),
                                        sb(d["base"].astype(f)), orc.split_batches(d["base"].astype(f), c.S)[-1])
    assert vs.dtype == f and tpt.grad.dtype == (torch.float64 if prec == "f64" else torch.float32)
    return dict(vs=vs.T, pg=pg.T, dl=tpt.grad.numpy(), db=bt.grad.numpy(), loss=float(loss.detach()))


class _VtraceRun:
    """the kernel's inputs on the device, and calls into output buffers pre-filled with NaN"""

    def __init__(self, xb, c, d):
        self.lib, self.c = xb["lib"], c
        self.inp = [dev(d["tp"]), dev(d["base"]), dev(d["bp"]), dev(d["act"]), dev(d["done"].view(np.uint8)), dev(d["rew"])]

    def __call__(self, with_vs_pg=True, loss0=0.0, inp=None):
        from xingtian_b200.engine import _ptr, stream_ptr
        c, N = self.c, self.c.k * self.c.S
        nan = lambda *shape: torch.full(shape, float("nan"), device="cuda")  # noqa: E731
        out = dict(dl=nan(N, c.A), db=nan(N), vs=nan(N) if with_vs_pg else None, pg=nan(N) if with_vs_pg else None,
                   loss=torch.full((1,), loss0, device="cuda"))
        ptrs = [_ptr(t) for t in (inp or self.inp)]
        rc = self.lib.xtb_vtrace_loss_grad(*ptrs, c.k, c.S, c.A, c.gamma, _ptr(out["dl"]), _ptr(out["db"]), _ptr(out["vs"]),
                                           _ptr(out["pg"]), _ptr(out["loss"]), stream_ptr())
        assert rc == 0, self.lib.xtb_last_error()
        torch.cuda.synchronize()
        return {k: (v.cpu().numpy() if v is not None else None) for k, v in out.items()}


@pytest.mark.parametrize("c", VTRACE, ids=[c.id for c in VTRACE])
def test_vtrace_kernel_against_float64(xb, c):
    """vs and pg_adv on the kept rows, the gradients on every row and the loss: max-norm error from float64 at most 4x
    that of the fp32 oracle + VT_FLOOR; then the output contract"""
    d = _vtrace_data(c)
    _assert_regimes(c, d)
    r64, r32 = _vtrace_reference(c, d, "f64"), _vtrace_reference(c, d, "f32")
    run = _VtraceRun(xb, c, d)
    got = run()
    k, S, T = c.k, c.S, c.S - 1
    gv = dict(vs=got["vs"].reshape(k, S)[:, :T], pg=got["pg"].reshape(k, S)[:, :T], dl=got["dl"], db=got["db"],
              loss=got["loss"][0])
    errs = {q: (rel_err(gv[q], r64[q]), rel_err(r32[q], r64[q])) for q in ("vs", "pg", "dl", "db", "loss")}
    record("vtrace_vs_f64/%s" % c.id, {q: ["%.2e" % a, "%.2e" % b] for q, (a, b) in errs.items()})
    bad = {q: e for q, e in errs.items() if not e[0] <= 4 * e[1] + VT_FLOOR}
    assert not bad, bad

    # every output written; row S - 1 exactly zero
    for q in ("dl", "db", "vs", "pg"):
        assert not np.isnan(got[q]).any(), q
    last = ~_kept(c)
    assert (got["dl"][last] == 0).all() and (got["db"][last] == 0).all()
    assert (got["vs"][last] == 0).all() and (got["pg"][last] == 0).all()
    # one block (k <= 4 warps) adds the loss with one atomic: bitwise reproducible; more blocks add in any order
    one_block = k <= 4

    def same_loss(a, b):
        return a == b if one_block else abs(a - b) <= 1e-6 * abs(b)

    # row S - 1's done, reward, action and both logit rows have no effect
    alt = {q: v.copy() for q, v in d.items()}
    alt["done"][last] = ~alt["done"][last]
    alt["rew"][last] += 3.0
    alt["act"][last] = (alt["act"][last] + 1) % c.A
    alt["tp"][last] = -alt["tp"][last] + 1.0
    alt["bp"][last] = alt["bp"][last] * 0.5 - 2.0
    moved = run(inp=_VtraceRun(xb, c, alt).inp)
    for q in ("dl", "db", "vs", "pg"):
        np.testing.assert_array_equal(moved[q], got[q], err_msg=q)
    assert same_loss(moved["loss"][0], got["loss"][0]), (moved["loss"][0], got["loss"][0])
    # vs / pg_adv are optional outputs (the learner passes NULL): the gradients do not change
    bare = run(with_vs_pg=False)
    np.testing.assert_array_equal(bare["dl"], got["dl"])
    np.testing.assert_array_equal(bare["db"], got["db"])
    # loss_out accumulates
    acc = run(loss0=1.5)
    want = np.float32(1.5) + np.float32(got["loss"][0])
    assert (acc["loss"][0] == want) if one_block else abs(acc["loss"][0] - want) <= 1e-6 * abs(want), (acc["loss"][0], want)


def test_vtrace_kernel_refuses_bad_arguments(xb):
    """n_traj 0, step_len 1, adim 0 and MAX_ADIM + 1 and each null pointer: XTB_ERR_ARG with a message, no launch"""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = xb["lib"]
    k, S, A = 2, 8, 4
    N = k * S
    # the logit and dlogits buffers hold MAX_ADIM columns: the accepted call below runs with adim = MAX_ADIM
    wide = lambda: dev(np.zeros((N, MAX_ADIM), np.float32))  # noqa: E731
    bufs = [wide(), dev(np.zeros(N, np.float32)), wide(), dev(np.zeros(N, np.int32)), dev(np.zeros(N, np.uint8)),
            dev(np.zeros(N, np.float32)), wide(), dev(np.zeros(N, np.float32)), dev(np.zeros(N, np.float32)),
            dev(np.zeros(N, np.float32)), dev(np.zeros(1, np.float32))]

    def call(n_traj=k, step_len=S, adim=A, null=None):
        p = [None if i == null else _ptr(t) for i, t in enumerate(bufs)]
        return lib.xtb_vtrace_loss_grad(*p[:6], n_traj, step_len, adim, 0.99, *p[6:], stream_ptr())

    torch.cuda.synchronize()
    before = lib.xtb_launch_count()
    sizes = [dict(n_traj=0), dict(step_len=1), dict(adim=0), dict(adim=MAX_ADIM + 1)]
    nulls = [dict(null=i) for i in (0, 1, 2, 3, 4, 5, 6, 7, 10)]      # every pointer but the optional vs / pg
    for i, kw in enumerate(nulls):        # alternate the two messages, so each refusal must write its own
        for kw, msg in ((sizes[i % len(sizes)], b"bad sizes"), (kw, b"null pointer")):
            assert call(**kw) == XTB_ERR_ARG, kw
            assert msg in lib.xtb_last_error() and b"xtb_vtrace_loss_grad" in lib.xtb_last_error(), kw
    assert lib.xtb_launch_count() == before
    assert call(null=8) == 0 and call(null=9) == 0 and call(adim=MAX_ADIM) == 0      # vs / pg optional; 32 actions
    assert lib.xtb_launch_count() == before + 3


# ---- b. the learner step against float64 ----------------------------------------------------------------------------
class LCase(collections.namedtuple("LCase", "F A k S act")):
    """F x F x 4 uint8 frames, A actions, k trajectories of S steps, ReLU (the product model) or tanh"""

    @property
    def id(self):
        return "F%d-A%d-k%d-S%d-%s" % (self.F, self.A, self.k, self.S, self.act)

    @property
    def n(self):
        return self.k * self.S


LEARNER = [
    LCase(84, 4, 4, 128, "relu"),         # the C3 benchmark's 512 samples
    LCase(84, 4, 4, 50, "relu"),          # the default sample_batch_step with BATCH_SIZE 200
    LCase(84, 18, 5, 33, "relu"), LCase(84, 4, 1, 2, "relu"),
    LCase(42, 4, 3, 50, "relu"), LCase(42, 18, 2, 129, "relu"),
    LCase(84, 4, 4, 50, "tanh"), LCase(84, 18, 5, 33, "tanh"),
]
HEADS = ("explore_agent/conv2d_3/kernel", "explore_agent/conv2d_3/bias", "explore_agent/dense/kernel",
         "explore_agent/dense/bias")


def _arch(c):
    arch = orc.impala_cnn_arch((c.F, c.F, 4), c.A)
    if c.act == "tanh":
        arch = dict(arch, layers=[(n, k, s, dict(sp, act=("tanh" if sp.get("act") == "relu" else sp.get("act"))))
                                  for n, k, s, sp in arch["layers"]])
    return arch


def _biased(w, seed):
    """non-zero biases: at their initial zeros every layer maps a zero row to zero, which hides a kernel that reads
    rows past the batch"""
    rng = np.random.default_rng(seed)
    return collections.OrderedDict((k, (v + 0.1 * rng.standard_normal(v.shape)).astype(np.float32) if k.endswith("/bias") else v)
                                   for k, v in w.items())


class _Learner:
    """the product ImpalaCnnOpt (ReLU) through Registers.model, or the tanh net with its global-clip-40 Adam, stepped
    through xtb_impala_train directly"""

    def __init__(self, c, lr=0.0, graph=False):
        import xingtian_b200  # noqa: F401
        from xingtian_b200 import capi
        from xingtian_b200.engine import Adam, Net
        from xingtian_b200.registry import Registers
        self.c, self.graph = c, graph
        if c.act == "relu":
            info = {"state_dim": [c.F, c.F, 4], "action_dim": c.A, "input_dtype": "uint8", "state_mean": 0.0,
                    "state_std": 255.0, "max_batch": c.n,
                    "model_config": {"LR": lr, "sample_batch_step": c.S, "grad_norm_clip": 40.0, "init_seed": 3,
                                     "use_cuda_graph": graph}}
            self.model = Registers.model["ImpalaCnnOpt"](info)
            self.net, self.opt = self.model.net, self.model.opt
            assert list(self.net.ptable) == list(orc.param_shapes(_arch(c)))
            self.net.set_weights(_biased(self.net.get_weights(), c.F + c.A))
        else:
            self.model = None
            arch = _arch(c)
            self.net = Net(arch, max_batch=c.n)
            self.net.set_weights(_biased(orc.init_weights(arch, seed=5, baseline_norm_std=0.01), c.F + c.A))
            self.opt = Adam(self.net, lr, eps=1e-8, clip_mode=capi.CLIP_GLOBAL_NORM, clip=40.0)
        self.loss = torch.zeros(1, device="cuda")

    def step(self, dd):
        """one learner step on the device data dd; returns the loss"""
        from xingtian_b200.capi import check
        from xingtian_b200.engine import _ptr, stream_ptr
        c = self.c
        if self.model is not None:
            self.model.use_graph = self.graph
            self.model.train_device(dd["obs"], dd["bp"], dd["act"], dd["done"], dd["rew"], c.n, self.loss)
        else:
            self.loss.zero_()
            net = self.net
            check(net.lib.xtb_impala_train(net.handle, self.opt.handle, _ptr(dd["obs"]), None, _ptr(dd["bp"]), _ptr(dd["act"]),
                                           _ptr(dd["done"]), _ptr(dd["rew"]), c.n, c.S, 0.99, net.tid["explore_agent/conv2d_3"],
                                           net.tid["explore_agent/dense"], _ptr(self.loss), 1 if self.graph else 0,
                                           stream_ptr()))
        torch.cuda.synchronize()
        return float(self.loss.cpu()[0])

    def grads(self):
        return self.net.get_weights(self.net.grads)


def _learner_data(c, w, rewards=None):
    """uint8 frames; behaviour logits = the fp32 oracle's logits + 0.5 N(0, 1); rewards N(0, 2); dones ~3 % plus one at
    T - 1 of trajectory 0 and one at its row S - 1"""
    rng = np.random.default_rng(c.F * 100 + c.A * 10 + c.n)
    obs = rng.integers(0, 256, (c.n, c.F, c.F, 4), dtype=np.uint8)
    with torch.no_grad():
        logits = orc.forward(_arch(c), w, obs)[0].numpy()
    bp = (logits + 0.5 * rng.standard_normal(logits.shape)).astype(np.float32)
    act = rng.integers(0, c.A, c.n).astype(np.int32)
    rew = (2 * rng.standard_normal(c.n) if rewards is None else rewards(rng, c.n)).astype(np.float32)
    done = rng.random(c.n) < 0.03
    done[c.S - 2] = done[c.S - 1] = True
    lsm = lambda x: x - x.max(-1, keepdims=True) - np.log(np.exp(x - x.max(-1, keepdims=True)).sum(-1, keepdims=True))  # noqa: E731
    pick = lambda x: np.take_along_axis(lsm(x.astype(np.float64)), act[:, None].astype(np.int64), 1)[:, 0]  # noqa: E731
    rho = np.exp(pick(logits) - pick(bp))[np.arange(c.n) % c.S != c.S - 1]
    return dict(obs=obs, bp=bp, act=act, done=done, rew=rew, rho=rho)


def _on_device(d):
    return dict(obs=dev(d["obs"]), bp=dev(d["bp"]), act=dev(d["act"]), done=dev(d["done"].view(np.uint8)), rew=dev(d["rew"]))


def _learner_oracle(c, w, d, prec, lr=0.0):
    with orc.precision(prec), np.errstate(over="ignore", under="ignore"):
        ref = orc.ImpalaLearner(_arch(c), w, lr=lr, grad_norm_clip=40.0, sample_batch_step=c.S, gamma=_f32(0.99))
        loss, g = ref.loss_and_grads(d["obs"], d["bp"], d["act"], d["done"], d["rew"])
        g = {k: t.detach().numpy().astype(np.float64) for k, t in zip(ref.names, g)}
    return float(loss.detach()), g, float(np.sqrt(sum(float((v ** 2).sum()) for v in g.values())))


_LEARNER_REF = {}   # case id -> weights, data and the float64 / fp32 oracle (independent of the kernel path)


def _learner_reference(c, w):
    if c.id not in _LEARNER_REF:
        d = _learner_data(c, w)
        _LEARNER_REF[c.id] = dict(w=w, d=d, f64=_learner_oracle(c, w, d, "f64"), f32=_learner_oracle(c, w, d, "f32"))
    return _LEARNER_REF[c.id]


@pytest.mark.parametrize("c", LEARNER, ids=[c.id for c in LEARNER])
def test_learner_step_against_float64(xb, tc_mode, c):
    """LR 0: the weights come back bitwise, and the loss, every parameter gradient (relative L2) and the global norm
    the optimiser computed are at most 4x torch-CPU fp32's distance from float64, + a floor of 6e-5 (tensor cores) or
    1e-5 (fp32) x max(1, sqrt(n / 128)), + the suite's ReLU flip allowance on the ReLU trunk's gradients"""
    lrn = _Learner(c)
    w0 = lrn.net.get_weights()
    ref = _learner_reference(c, w0)
    for k in w0:
        assert np.array_equal(w0[k], ref["w"][k]), k
    d = ref["d"]
    if c.n >= 64:
        assert (d["rho"] < 1).any() and (d["rho"] > 1).any()
    loss = lrn.step(_on_device(d))
    g = lrn.grads()
    gn = lrn.opt.grad_norm()
    w1 = lrn.net.get_weights()
    for k in w0:
        assert np.array_equal(w1[k], w0[k]), k
    (l64, g64, n64), (l32, g32, n32) = ref["f64"], ref["f32"]
    floor = (6e-5 if tc_mode == 1 else 1e-5) * max(1.0, np.sqrt(c.n / 128.0))
    flip = (RELU_FLIP_TC if tc_mode == 1 else RELU_FLIP_F32) if c.act == "relu" else 0.0
    errs = {k: (l2_rel(g[k], g64[k]), l2_rel(g32[k], g64[k])) for k in g64}
    errs["loss"] = (abs(loss - l64) / max(1.0, abs(l64)), abs(l32 - l64) / max(1.0, abs(l64)))
    errs["grad_norm"] = (abs(gn - n64) / n64, abs(n32 - n64) / n64)
    record("impala_step_vs_f64/%s/%s" % (c.id, "tcgen05" if tc_mode else "fp32"),
           {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in errs.items()})
    bad = {k: e for k, e in errs.items()
           if not e[0] <= 4 * e[1] + floor + (flip if k in g64 and k not in HEADS else 0.0)}
    assert not bad, bad


# ---- c. eager, graph capture, graph replay and the data-parallel path -----------------------------------------------
FORMS = [LCase(84, 4, 4, 50, "relu"), LCase(42, 4, 3, 50, "relu")]
FORMS_BOUND = 4e-6     # reordered fp32 sums, relative L2 per tensor (observed <= 4.3e-7 on an H100 80GB HBM3 at 700 W)


@pytest.mark.parametrize("c", FORMS, ids=[c.id for c in FORMS])
def test_learner_step_forms_agree(xb, tc_mode, c):
    """eager, eager again, the graph call that captures, a replay and eager with a one-rank communicator installed (the
    gradient all-reduce runs) at LR 0: the weights come back bitwise, the loss (block_atomic_add sums it in any block
    order) within 1e-6, the gradients of the layers that run on the tensor cores bitwise (their weight and bias
    gradients are ordered sums), and every other gradient tensor within FORMS_BOUND of the first eager call's
    (relative L2): the weight gradients of the dense heads, and of a conv layer that runs on the CUDA cores, add split-K
    partial sums with atomics, and colsum_kernel adds bias sums with atomics, so even two eager calls differ there in the
    last bits"""
    lib = xb["lib"]
    lrn = _Learner(c)
    w0 = lrn.net.get_weights()
    dd = _on_device(_learner_reference(c, w0)["d"])
    out = {}
    out["eager"] = (lrn.step(dd), lrn.grads())
    out["eager_again"] = (lrn.step(dd), lrn.grads())
    lrn.graph = True
    c0, r0 = lib.xtb_graph_capture_count(), lib.xtb_graph_replay_count()
    out["capture"] = (lrn.step(dd), lrn.grads())
    assert (lib.xtb_graph_capture_count() - c0, lib.xtb_graph_replay_count() - r0) == (1, 1)
    out["replay"] = (lrn.step(dd), lrn.grads())
    assert (lib.xtb_graph_capture_count() - c0, lib.xtb_graph_replay_count() - r0) == (1, 2)
    lrn.graph = False
    with one_rank_comm():
        out["one_rank_comm"] = (lrn.step(dd), lrn.grads())
    w1 = lrn.net.get_weights()
    for k in w0:
        assert np.array_equal(w1[k], w0[k]), k
    le, ge = out["eager"]
    on_tc = [n for i, (n, _, _, _) in enumerate(lrn.net.arch["layers"]) if tc_mode == 1 and lrn.net.layer_plan(i)["tc"]]
    exact = {n + sfx for n in on_tc for sfx in ("/kernel", "/bias")}
    assert exact or tc_mode == 0
    errs = {form: {k: l2_rel(g[k], ge[k]) for k in ge} for form, (_, g) in out.items()}
    record("impala_step_forms/%s/%s" % (c.id, "tcgen05" if tc_mode else "fp32"),
           {"loss": {form: "%.9g" % l for form, (l, _) in out.items()}, "bitwise": sorted(exact),
            "grad_l2_rel_to_eager": {form: {k: "%.1e" % e for k, e in es.items() if e > 0} for form, es in errs.items()}})
    for form, (l, g) in out.items():
        assert abs(l - le) <= 1e-6 * abs(le), (form, l, le)
        bad = {k: e for k, e in errs[form].items() if not (e == 0.0 if k in exact else e <= FORMS_BOUND)}
        assert not bad, (form, bad)
        for k in exact:
            np.testing.assert_array_equal(g[k], ge[k], err_msg="%s %s" % (form, k))


# ---- d. the clip and Adam wiring ------------------------------------------------------------------------------------
def test_learner_step_clips_the_global_norm_and_takes_one_adam_step(xb, tc_mode):
    """LR 5e-4 with rewards mostly +1 (clipped): the summed losses give a global norm far above the clip 40.
    - The norm the optimiser computed is the float64 norm of the device's own gradient within 1e-5: the reported norm
      is |grad_scale| times the norm of every parameter's gradient, so a wrong grad_scale or a parameter left out
      shows here.
    - The clip: after the first step Adam's moments are (1 - beta1) g' and (1 - beta2) g'^2 of the clipped gradient
      g' = g * 40 / norm, within 1e-6 relative L2 of clip_by_global_norm(g, 40) in float64 (the betas as the device
      holds them, in fp32).  The update alone barely shows the clip: the first Adam step is close to lr * sign(g).
    - The update is one TFAdam step of the clipped gradient in float64, within 1e-5 relative L2 (against the float64
      weights rounded to fp32, as the device stores them)."""
    c = LCase(84, 4, 4, 128, "relu")
    lr = 5e-4
    lrn = _Learner(c, lr=lr)
    w0 = lrn.net.get_weights()
    d = _learner_data(c, w0, rewards=lambda rng, n: 1.0 + 0.5 * rng.standard_normal(n))
    lrn.step(_on_device(d))
    g = lrn.grads()
    gn = lrn.opt.grad_norm()
    w1 = lrn.net.get_weights()
    names = list(w0)
    with orc.precision("f64"):
        gl = [torch.from_numpy(g[k].astype(np.float64)) for k in names]
        clipped, n64 = orc.clip_by_global_norm(gl, 40.0)
        params = [torch.from_numpy(w0[k].astype(np.float64)) for k in names]
        orc.TFAdam(params, lr, eps=1e-8).step(clipped)
    upd = np.concatenate([(w1[k].astype(np.float64) - w0[k]).ravel() for k in names])
    want = np.concatenate([(p.numpy().astype(np.float32).astype(np.float64) - w0[k]).ravel() for k, p in zip(names, params)])
    err = l2_rel(upd, want)
    b1, b2 = 1.0 - _f32(0.9), 1.0 - _f32(0.999)
    mom = lrn.net.get_weights(lrn.opt.m)
    var = lrn.net.get_weights(lrn.opt.v)
    cl = np.concatenate([t.numpy().ravel() for t in clipped])
    m_err = l2_rel(np.concatenate([mom[k].ravel() for k in names]), b1 * cl)
    v_err = l2_rel(np.concatenate([var[k].ravel() for k in names]), b2 * cl * cl)
    record("impala_step_clip_adam/%s" % ("tcgen05" if tc_mode else "fp32"),
           {"grad_norm": "%.6g" % gn, "norm_rel_err": "%.2e" % (abs(gn - n64) / n64), "m_l2_rel": "%.2e" % m_err,
            "v_l2_rel": "%.2e" % v_err, "update_l2_rel": "%.2e" % err})
    assert n64 > 40.0 * 10, n64
    assert abs(gn - n64) <= 1e-5 * n64, (gn, n64)
    assert m_err <= 1e-6 and v_err <= 1e-6, (m_err, v_err)
    assert err <= 1e-5, err
