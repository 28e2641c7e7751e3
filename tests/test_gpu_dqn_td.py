"""DQN's TD learner step (DqnCnn / DqnMlp through xtb_dqn_train and xtb_dqn_train_weighted) against float64:

a. dqn_loss_kernel through xtb_dqn_td_loss_grad: the TD target y, |TD error|, dq and the loss against the oracle's float64
   target and autograd, at batches around the kernel's 128-thread blocks, one to 18 actions, gamma 0 and 1, plain and
   double DQN, the squared error and Huber, n-step discounts, ring indices and per-sample weights; each case asserts
   the data regimes it is named for.  Its contract: every dq entry written and zero off the taken action, y / td_abs
   optional, the loss accumulated, bad arguments refused without a launch.  xtb_mse_loss_grad the same way;
b. the learner step at LR 0: the loss, td_abs, every parameter gradient and the global norm the optimiser saw, against
   float64 on both kernel paths, for each fused dueling instantiation, the layer path and every TD form, with a target
   net whose weights differ from the online net's;
c. the step's forms: eager, graph capture, graph replay and the data-parallel path with a one-rank communicator;
d. the per-tensor clip and Adam wiring of one DqnCnn step, and one unclipped DqnMlp step.

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
# a few fp32 ulps on top of 4 x the fp32 oracle's distance from float64 (observed on an H100 80GB HBM3 at 700 W: at most
# 7.5 % of the bound, on the MSE kernel's loss at B = 1000, A = 18; the TD kernel at most 6 %, on dq of the 1000-sample
# Huber case)
TD_FLOOR = 2e-6


def _f32(x):
    """the value a C float argument carries"""
    return float(np.float32(x))


@pytest.fixture(autouse=True)
def _restore_dqn_config():
    """import_config writes HIDDEN_SIZE / NUM_LAYERS / LR into xingtian_b200.model.dqn's globals: restore them"""
    from xingtian_b200.model import dqn as model_mod
    saved = {k: v for k, v in vars(model_mod).items() if k.isupper()}
    yield
    for k in [k for k in vars(model_mod) if k.isupper() and k not in saved]:
        delattr(model_mod, k)
    for k, v in saved.items():
        setattr(model_mod, k, v)


# ---- a. xtb_dqn_td_loss_grad ----------------------------------------------------------------------------------------
class KCase(collections.namedtuple("KCase", "B A gamma double huber disc idx wt")):
    """B samples, A actions; double: qn_o given; huber: delta (0 = squared error); disc: per-row n-step discounts;
    idx: rows of a ring of B + 7 indexed through idx; wt: per-sample weights"""

    @property
    def id(self):
        f = [n for n, on in (("double", self.double), ("disc", self.disc), ("idx", self.idx), ("wt", self.wt)) if on]
        return "B%d-A%d-g%g-%s%s" % (self.B, self.A, self.gamma, "huber%g" % self.huber if self.huber else "mse",
                                     "".join("-" + x for x in f))

    @property
    def rows(self):
        return self.B + 7 if self.idx else self.B


TD = [
    # the shapes of the fp32-oracle test this replaces: (B, A, double) = (32, 4, no), (512, 4, no), (32, 6, yes)
    KCase(32, 4, 0.99, False, 0.0, False, False, False), KCase(512, 4, 0.99, False, 0.0, False, False, False),
    KCase(32, 6, 0.99, True, 0.0, False, False, False),
    # one sample, one action; one sample of a ring with every option
    KCase(1, 1, 0.99, False, 0.0, False, False, False), KCase(1, 4, 0.99, True, 1.0, True, True, True),
    # 127 / 128 / 129: a partly filled, a full and a second block of 128 threads
    KCase(127, 2, 0.99, True, 1.0, True, True, True), KCase(128, 4, 1.0, False, 1.0, False, True, False),
    KCase(129, 6, 0.0, True, 0.0, True, False, True), KCase(129, 1, 0.99, False, 1.0, False, True, True),
    KCase(128, 18, 0.99, True, 0.0, False, False, False), KCase(127, 6, 1.0, False, 0.0, True, False, False),
    KCase(1000, 18, 0.99, True, 0.5, True, True, True), KCase(1000, 2, 0.0, False, 0.0, False, True, False),
    # 4097: 33 blocks, the last with one sample
    KCase(4097, 4, 0.99, False, 0.0, True, True, True), KCase(4097, 18, 1.0, True, 1.0, False, False, True),
]


def _td_data(c):
    """q / qn_t / qn_o [B, A] by sample; action / reward / done / disc [rows] by ring row, read through idx"""
    rng = np.random.default_rng(c.B * 100 + c.A * 10 + int(c.huber * 4))
    B, A, N = c.B, c.A, c.rows
    q = rng.standard_normal((B, A)).astype(np.float32)
    qt = rng.standard_normal((B, A)).astype(np.float32)
    qo = rng.standard_normal((B, A)).astype(np.float32)
    act = rng.integers(0, A, N).astype(np.int32)
    rew = (3 * rng.standard_normal(N)).astype(np.float32)           # TD errors mostly beyond a Huber delta of 1
    done = rng.random(N) < 0.15
    disc = np.where(done, 0.0, np.float32(0.99) ** rng.integers(1, 4, N)).astype(np.float32)
    disc[3::11] = 0.0                                                # windows that hit a terminal step, rows not done
    idx = rng.integers(0, N, B).astype(np.int32) if c.idx else np.arange(B, dtype=np.int32)
    if c.idx and B > 1:
        idx[-1] = N - 1                                              # the ring's last row
        idx[B // 2] = idx[0]                                         # a repeated row
    elif c.idx:
        idx[0] = N - 1
    r = idx
    if A >= 2:
        # tied online maxima whose target values differ, on rows that bootstrap
        for b in range(0, B, 5):
            i, j = sorted(rng.choice(A, 2, replace=False))
            qo[b, i] = qo[b, j] = qo[b].max() + 0.5
            qt[b, j] = qt[b, i] + 0.75
            done[r[b]] = False
            disc[r[b]] = np.float32(0.99)
    if c.huber and B >= 4:
        # TD errors of exactly +delta and -delta: done rows with y = reward
        for b, s in ((1, 1.0), (2, -1.0)):
            done[r[b]], rew[r[b]] = True, 0.5
            q[b, act[r[b]]] = 0.5 + s * c.huber
    wt = rng.uniform(0.0, 2.0, B).astype(np.float32)
    wt[::9] = 0.0
    return dict(q=q, qt=qt, qo=qo, act=act, rew=rew, done=done, disc=disc, idx=idx, wt=wt)


def _assert_td_regimes(c, d):
    """each regime the case is named for occurs on the rows the kernel reads"""
    r = d["idx"]
    done, disc = d["done"][r], d["disc"][r]
    if c.B < 32:
        return
    assert done.any() and not done.all()
    if c.disc:
        assert ((disc == 0) & ~done).any()
    if c.double and c.A >= 2:
        tied = [b for b in range(c.B) if (d["qo"][b] == d["qo"][b].max()).sum() > 1 and not done[b]]
        assert tied and all(d["qt"][b, np.argmax(d["qo"][b])] != d["qt"][b, c.A - 1 - np.argmax(d["qo"][b][::-1])] for b in tied)
    if c.huber:
        y = _td_reference(c, d, "f64")["y"]
        diff = d["q"][np.arange(c.B), d["act"][r]].astype(np.float64) - y
        assert (np.abs(diff) > c.huber).any() and (np.abs(diff) < c.huber).any()
        assert (diff == c.huber).any() and (diff == -c.huber).any()
    if c.idx:
        assert len(np.unique(r)) < c.B and (r == c.rows - 1).any()
    if c.wt:
        assert (d["wt"] == 0).any()


def _td_reference(c, d, prec):
    """y and |TD error| [B], d loss / d q [B, A] and the loss, in `prec`"""
    f = np.float64 if prec == "f64" else np.float32
    r = d["idx"]
    a = d["act"][r].astype(np.int64)
    with orc.precision(prec):
        y = orc.dqn_targets(d["q"].astype(f), d["qt"].astype(f), d["act"][r], d["rew"][r], d["done"][r], _f32(c.gamma),
                            d["qo"].astype(f) if c.double else None, d["disc"][r] if c.disc else None)
    assert y.dtype == f
    qt = torch.from_numpy(d["q"].astype(f)).requires_grad_(True)
    diff = qt - torch.from_numpy(y)
    if c.huber > 0:
        ad = diff.abs()
        per = torch.where(ad <= c.huber, 0.5 * diff * diff, c.huber * (ad - 0.5 * c.huber))
    else:
        per = diff * diff
    if c.wt:
        per = per * torch.from_numpy(d["wt"].astype(f))[:, None]
    loss = per.mean()
    loss.backward()
    rows = np.arange(c.B)
    return dict(y=y[rows, a], td=np.abs(diff.detach().numpy()[rows, a]), dq=qt.grad.numpy(), loss=float(loss.detach()))


class _TdRun:
    """the kernel's inputs on the device, and calls into output buffers pre-filled with NaN"""

    def __init__(self, xb, c, d):
        self.lib, self.c, self.d = xb["lib"], c, d
        self.inp = dict(q=dev(d["q"]), qt=dev(d["qt"]), qo=dev(d["qo"]), idx=dev(d["idx"]), act=dev(d["act"]), rew=dev(d["rew"]),
                        done=dev(d["done"].view(np.uint8)), disc=dev(d["disc"]), wt=dev(d["wt"]))

    def __call__(self, with_y_td=True, loss0=0.0):
        from xingtian_b200.engine import _ptr, stream_ptr
        c, i = self.c, self.inp
        nan = lambda *shape: torch.full(shape, float("nan"), device="cuda")  # noqa: E731
        out = dict(dq=nan(c.B, c.A), y=nan(c.B) if with_y_td else None, td=nan(c.B) if with_y_td else None,
                   loss=torch.full((1,), loss0, device="cuda"))
        opt = lambda on, t: _ptr(t) if on else None  # noqa: E731
        rc = self.lib.xtb_dqn_td_loss_grad(_ptr(i["q"]), _ptr(i["qt"]), opt(c.double, i["qo"]), opt(c.idx, i["idx"]), _ptr(i["act"]),
                                           _ptr(i["rew"]), _ptr(i["done"]), opt(c.disc, i["disc"]), c.B, c.A, c.gamma, c.huber,
                                           1.0 / (c.B * c.A), opt(c.wt, i["wt"]), _ptr(out["dq"]), _ptr(out["y"]), _ptr(out["td"]),
                                           _ptr(out["loss"]), stream_ptr())
        assert rc == 0, self.lib.xtb_last_error()
        torch.cuda.synchronize()
        return {k: (v.cpu().numpy() if v is not None else None) for k, v in out.items()}

    def legacy(self):
        """the same step through xtb_dqn_loss_grad, the entry without idx, disc, Huber, weights and td_abs"""
        from xingtian_b200.engine import _ptr, stream_ptr
        c, i = self.c, self.inp
        assert not (c.idx or c.disc or c.huber or c.wt)
        out = dict(dq=torch.full((c.B, c.A), float("nan"), device="cuda"), y=torch.full((c.B,), float("nan"), device="cuda"),
                   loss=torch.zeros(1, device="cuda"))
        rc = self.lib.xtb_dqn_loss_grad(_ptr(i["q"]), _ptr(i["qt"]), _ptr(i["qo"]) if c.double else None, _ptr(i["act"]), _ptr(i["rew"]),
                                        _ptr(i["done"]), c.B, c.A, c.gamma, 1.0 / (c.B * c.A), _ptr(out["dq"]), _ptr(out["y"]),
                                        _ptr(out["loss"]), stream_ptr())
        assert rc == 0, self.lib.xtb_last_error()
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("c", TD, ids=[c.id for c in TD])
def test_td_kernel_against_float64(xb, c):
    """y, |TD error| and dq (max-norm) and the loss: error from float64 at most 4x that of the fp32 oracle + TD_FLOOR;
    then the output contract"""
    d = _td_data(c)
    _assert_td_regimes(c, d)
    r64, r32 = _td_reference(c, d, "f64"), _td_reference(c, d, "f32")
    run = _TdRun(xb, c, d)
    got = run()
    gv = dict(y=got["y"], td=got["td"], dq=got["dq"], loss=got["loss"][0])
    errs = {k: (rel_err(gv[k], r64[k]), rel_err(r32[k], r64[k])) for k in ("y", "td", "dq")}
    errs["loss"] = (abs(gv["loss"] - r64["loss"]) / max(1.0, abs(r64["loss"])), abs(r32["loss"] - r64["loss"]) / max(1.0, abs(r64["loss"])))
    record("dqn_td_vs_f64/%s" % c.id, {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in errs.items()})
    bad = {k: e for k, e in errs.items() if not e[0] <= 4 * e[1] + TD_FLOOR}
    assert not bad, bad

    # every output written; dq exactly zero off the taken action
    for k in ("dq", "y", "td"):
        assert not np.isnan(got[k]).any(), k
    taken = np.eye(c.A, dtype=bool)[d["act"][d["idx"]]]
    assert (got["dq"][~taken] == 0).all()
    # one block adds the loss with one atomic: bitwise reproducible; more blocks add in any order
    one_block = c.B <= 128

    def same_loss(a, b):
        return a == b if one_block else abs(a - b) <= 1e-6 * abs(b)

    # y / td_abs are optional outputs: dq and the loss do not change
    bare = run(with_y_td=False)
    np.testing.assert_array_equal(bare["dq"], got["dq"])
    assert same_loss(bare["loss"][0], got["loss"][0])
    # loss_out accumulates
    acc = run(loss0=1.5)
    want = np.float32(1.5) + np.float32(got["loss"][0])
    assert same_loss(acc["loss"][0], want), (acc["loss"][0], want)
    # the reference-mode entry xtb_dqn_loss_grad forwards to the same kernel: the same dq, y and loss
    if not (c.idx or c.disc or c.huber or c.wt):
        old = run.legacy()
        np.testing.assert_array_equal(old["dq"], got["dq"])
        np.testing.assert_array_equal(old["y"], got["y"])
        assert same_loss(old["loss"][0], got["loss"][0]), (old["loss"][0], got["loss"][0])


def test_td_kernel_refuses_bad_arguments(xb):
    """batch 0, adim 0 and each required null pointer: XTB_ERR_ARG with a message, no launch; qn_o, idx, disc, wt, y and
    td_abs are optional"""
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = xb["lib"]
    B, A = 8, 4
    f = lambda *s: dev(np.zeros(s, np.float32))  # noqa: E731
    bufs = [f(B, A), f(B, A), f(B, A), dev(np.zeros(B, np.int32)), dev(np.zeros(B, np.int32)), f(B), dev(np.zeros(B, np.uint8)),
            f(B), f(B), f(B, A), f(B), f(B), f(1)]
    opt_ix = (2, 3, 7, 8, 10, 11)               # qn_o, idx, disc, wt, y_out, td_abs

    def call(batch=B, adim=A, null=()):
        p = [None if i in null else _ptr(t) for i, t in enumerate(bufs)]
        return lib.xtb_dqn_td_loss_grad(*p[:8], batch, adim, 0.99, 0.0, 1.0 / (B * A), *p[8:], stream_ptr())

    torch.cuda.synchronize()
    before = lib.xtb_launch_count()
    sizes = [dict(batch=0), dict(adim=0), dict(batch=-1)]
    nulls = [dict(null=(i,)) for i in (0, 1, 4, 5, 6, 9, 12)]     # q, qn_t, action, reward, done, dq, loss_out
    for i, null_kw in enumerate(nulls):   # alternate the two messages, so each refusal must write its own
        for kw, msg in ((sizes[i % len(sizes)], b"bad sizes"), (null_kw, b"null pointer")):
            assert call(**kw) == XTB_ERR_ARG, kw
            assert msg in lib.xtb_last_error() and b"xtb_dqn_td_loss_grad" in lib.xtb_last_error(), kw
    assert lib.xtb_launch_count() == before
    assert call(null=opt_ix) == 0 and call() == 0
    assert lib.xtb_launch_count() == before + 2


MSE = [(1, 1), (127, 4), (128, 6), (129, 2), (1000, 18), (4097, 4)]


@pytest.mark.parametrize("B,A", MSE, ids=["B%d-A%d" % s for s in MSE])
def test_mse_kernel_against_float64(xb, B, A):
    """Keras train_on_batch(state, y) with 'mse': dq = 2 (q - y) / (B A) and the loss against float64 (4x the fp32
    error + TD_FLOOR), every dq entry written, the loss accumulated"""
    from xingtian_b200.engine import _ptr, stream_ptr
    rng = np.random.default_rng(B * 10 + A)
    q = rng.standard_normal((B, A)).astype(np.float32)
    y = (q + 2 * rng.standard_normal((B, A))).astype(np.float32)
    y[::3] = q[::3]                                                    # rows with zero error
    ref = {}
    for prec, f in (("f64", torch.float64), ("f32", torch.float32)):
        qt = torch.from_numpy(q).to(f).requires_grad_(True)
        loss = ((qt - torch.from_numpy(y).to(f)) ** 2).mean()
        loss.backward()
        ref[prec] = (qt.grad.numpy(), float(loss.detach()))
    qd, yd = dev(q), dev(y)

    def run(loss0):
        dq = torch.full((B, A), float("nan"), device="cuda")
        lo = torch.full((1,), loss0, device="cuda")
        xb["capi"].check(xb["lib"].xtb_mse_loss_grad(_ptr(qd), _ptr(yd), B, A, 1.0 / (B * A), _ptr(dq), _ptr(lo), stream_ptr()))
        return dq.cpu().numpy(), float(lo.cpu()[0])

    got_dq, got_l = run(0.0)
    assert not np.isnan(got_dq).any()
    errs = {"dq": (rel_err(got_dq, ref["f64"][0]), rel_err(ref["f32"][0], ref["f64"][0])),
            "loss": (abs(got_l - ref["f64"][1]) / max(1.0, ref["f64"][1]), abs(ref["f32"][1] - ref["f64"][1]) / max(1.0, ref["f64"][1]))}
    record("mse_vs_f64/B%d-A%d" % (B, A), {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in errs.items()})
    bad = {k: e for k, e in errs.items() if not e[0] <= 4 * e[1] + TD_FLOOR}
    assert not bad, bad
    # loss_out accumulates (one block of 128 threads adds its sum with one atomic: bitwise; more blocks in any order)
    acc_dq, acc = run(0.75)
    np.testing.assert_array_equal(acc_dq, got_dq)
    want = float(np.float32(0.75) + np.float32(got_l))
    assert (acc == want) if B * A <= 128 else abs(acc - want) <= 1e-6 * want, (acc, want)


# ---- b. the learner step against float64 ----------------------------------------------------------------------------
class LCase(collections.namedtuple("LCase", "kind A B dueling hidden layers double huber nstep wt fuse plan")):
    """DqnCnn (84 x 84 x 4 frames, hidden 256) or DqnMlp (8 floats, `layers` ReLU layers of `hidden`); `plan`: the
    heads_kernel entry (kpl, amax) the step launches, (0, 0) layer by layer"""

    @property
    def id(self):
        f = [n for n, on in (("dueling", self.dueling), ("double", self.double), ("huber", self.huber), ("nstep", self.nstep),
                             ("wt", self.wt), ("nofuse", not self.fuse)) if on]
        net = "cnn" if self.kind == "cnn" else "mlp%dx%d" % (self.layers, self.hidden)
        return "%s-A%d-B%d-%s-%s" % (net, self.A, self.B, "fused%dx%d" % self.plan if self.plan[0] else "layers", "-".join(f) or "plain")


def _L(kind, A, B, dueling=False, hidden=256, layers=1, double=False, huber=False, nstep=False, wt=False, fuse=True, plan=(0, 0)):
    return LCase(kind, A, B, dueling, hidden, layers, double, huber, nstep, wt, fuse, plan)


LEARNER = [
    _L("cnn", 4, 1), _L("cnn", 4, 37, huber=True, wt=True), _L("cnn", 4, 512),
    _L("cnn", 18, 64), _L("cnn", 18, 64, double=True, nstep=True),
    _L("cnn", 4, 37, dueling=True, double=True, huber=True, plan=(8, 4)),
    _L("cnn", 6, 37, dueling=True, nstep=True, wt=True, plan=(8, 8)),
    _L("cnn", 9, 37, dueling=True, double=True, huber=True, nstep=True, wt=True),
    _L("cnn", 4, 37, dueling=True, fuse=False),
    _L("mlp", 8, 37, dueling=True, hidden=64, double=True, plan=(2, 8)),
    _L("mlp", 4, 37, dueling=True, hidden=128, huber=True, wt=True, plan=(8, 4)),
    _L("mlp", 6, 37, dueling=True, hidden=128, plan=(8, 8)),
    _L("mlp", 4, 1056, dueling=True, hidden=128, nstep=True, plan=(8, 4)),
    _L("mlp", 4, 1057, dueling=True, hidden=128, plan=(8, 4)),
    _L("mlp", 4, 4096, dueling=True, hidden=128, huber=True, nstep=True, wt=True, plan=(8, 4)),
    _L("mlp", 4, 37, dueling=True, hidden=512, plan=(16, 4)),
    _L("mlp", 6, 37, dueling=True, hidden=512, double=True, plan=(0, 0)),
    _L("mlp", 4, 133, hidden=128, layers=2, huber=True),
    _L("mlp", 4, 133, dueling=True, hidden=128, layers=2, double=True, nstep=True, wt=True, plan=(8, 4)),
]
HUBER = 1.0


def _heads(c):
    """the parameter tensors of the Q head (and the dueling adv head): no ReLU kink between them and the loss"""
    last = 1 if c.kind == "cnn" else c.layers
    names = ["dense_%d" % last] + (["dense_%d" % (last + 1)] if c.dueling else [])
    return {n + s for n in names for s in ("/kernel", "/bias")}


def _biased(w, seed):
    """non-zero biases: at their initial zeros every layer maps a zero row to zero, which hides a kernel that reads
    rows past the batch"""
    rng = np.random.default_rng(seed)
    return collections.OrderedDict((k, (v + 0.1 * rng.standard_normal(v.shape)).astype(np.float32) if k.endswith("/bias") else v)
                                   for k, v in w.items())


class _Learner:
    """an online and a target DqnCnn / DqnMlp with different weights, stepped through train_td_device"""

    def __init__(self, c, lr=0.0, graph=False):
        from xingtian_b200.model.dqn import DqnCnn, DqnMlp
        self.c = c
        cls, sd = (DqnCnn, [84, 84, 4]) if c.kind == "cnn" else (DqnMlp, [8])
        mk = lambda seed: cls({"state_dim": sd, "action_dim": c.A, "max_batch": c.B,  # noqa: E731
                               "model_config": {"dueling": c.dueling, "init_seed": seed, "LR": lr, "HIDDEN_SIZE": c.hidden,
                                                "NUM_LAYERS": c.layers, "use_cuda_graph": graph}})
        self.model, self.target = mk(7), mk(8)
        self.model.net.set_weights(_biased(self.model.net.get_weights(), c.A + c.B))
        self.target.net.set_weights(_biased(self.target.net.get_weights(), c.A + c.B + 1))
        self.net, self.opt = self.model.net, self.model.opt
        self.loss = torch.zeros(1, device="cuda")
        self.td = torch.zeros(c.B, device="cuda")

    def step(self, dd, plain=False):
        """one TD step on the device data dd; returns the loss and td_abs (None with plain: the unweighted entry)"""
        c = self.c
        self.model.train_td_device(self.target, dd["s"], dd["a"], dd["r"], dd["s2"], dd["d"], c.B, 0.99, self.loss, double_dqn=c.double,
                                   idx=dd["idx"], disc=dd["disc"] if c.nstep else None, huber_delta=HUBER if c.huber else 0.0,
                                   weights=dd["wt"] if c.wt else None, td_abs=None if plain else self.td)
        torch.cuda.synchronize()
        return float(self.loss.cpu()[0]), (None if plain else self.td.cpu().numpy())

    def grads(self):
        return self.net.get_weights(self.net.grads)


def _learner_data(c, rewards=3.0):
    """a ring of B + 5 transitions read through idx (a repeated row and the ring's last row); rewards N(0, rewards^2)"""
    rng = np.random.default_rng(c.A * 1000 + c.B)
    N = c.B + 5
    if c.kind == "cnn":
        s = rng.integers(0, 256, (N, 84, 84, 4), dtype=np.uint8)
        s2 = rng.integers(0, 256, (N, 84, 84, 4), dtype=np.uint8)
    else:
        s = rng.standard_normal((N, 8)).astype(np.float32)
        s2 = rng.standard_normal((N, 8)).astype(np.float32)
    idx = rng.integers(0, N, c.B).astype(np.int32)
    idx[-1] = N - 1
    if c.B > 2:
        idx[1] = idx[0]
    done = rng.random(N) < 0.1
    done[idx[c.B // 2]] = True
    disc = np.where(done, 0.0, np.float32(0.99) ** rng.integers(1, 4, N)).astype(np.float32)
    wt = rng.uniform(0.0, 2.0, c.B).astype(np.float32)
    wt[::7] = 0.0
    return dict(s=s, s2=s2, a=rng.integers(0, c.A, N).astype(np.int32), r=(rewards * rng.standard_normal(N)).astype(np.float32),
                d=done, disc=disc, idx=idx, wt=wt)


def _on_device(d):
    return dict(s=dev(d["s"]), s2=dev(d["s2"]), a=dev(d["a"]), r=dev(d["r"]), d=dev(d["d"].view(np.uint8)), disc=dev(d["disc"]),
                idx=dev(d["idx"]), wt=dev(d["wt"]))


def _oracle(c, arch, w, wt, d, prec):
    """the loss, td_abs, the gradients (float64 arrays) and their global norm, in `prec`; in float64 with double DQN also
    the online and the target net's Q(s') rows"""
    i = d["idx"]
    clip = 10.0 if c.kind == "cnn" else None
    with orc.precision(prec):
        ref = orc.DqnLearner(arch, w, lr=0.0, clipnorm=clip, gamma=_f32(0.99), double_dqn=c.double, target_weights=wt)
        loss, g, _, td = ref.loss_and_grads(d["s"][i], d["a"][i], d["r"][i], d["s2"][i], d["d"][i],
                                            disc=d["disc"][i] if c.nstep else None, huber=HUBER if c.huber else 0.0,
                                            weights=d["wt"] if c.wt else None)
        g = {k: t.detach().numpy().astype(np.float64) for k, t in zip(ref.names, g)}
        qn = ref.predict(d["s2"][i]) if c.double and prec == "f64" else None
        qt = ref.predict(d["s2"][i], target=True) if c.double and prec == "f64" else None
    return dict(loss=float(loss.detach()), g=g, td=td.astype(np.float64), norm=float(np.sqrt(sum(float((v ** 2).sum()) for v in g.values()))),
                qn=qn, qt=qt)


_LEARNER_REF = {}   # case id -> weights, data and the float64 / fp32 oracle (independent of the kernel path)


def _learner_reference(c, lrn):
    if c.id not in _LEARNER_REF:
        w, wt = lrn.net.get_weights(), lrn.target.net.get_weights()
        d = _learner_data(c)
        arch = lrn.model.arch
        assert list(w) == list(orc.param_shapes(arch))
        _LEARNER_REF[c.id] = dict(w=w, wt=wt, d=d, f64=_oracle(c, arch, w, wt, d, "f64"), f32=_oracle(c, arch, w, wt, d, "f32"))
    return _LEARNER_REF[c.id]


def _assert_learner_regimes(c, ref):
    d, r64 = ref["d"], ref["f64"]
    i = d["idx"]
    assert any(not np.array_equal(ref["w"][k], ref["wt"][k]) for k in ref["w"])       # the target net is its own
    if c.B >= 32:
        assert d["d"][i].any() and not d["d"][i].all()
        assert len(np.unique(i)) < c.B and (i == c.B + 4).any()
    if c.huber and c.B >= 32:
        assert (r64["td"] > HUBER).any() and (r64["td"] < HUBER).any()
    if c.wt:
        assert (d["wt"] == 0).any()
    if c.double:
        # the online argmax over Q(s') has no near-tie, which the device's rounding could resolve the other way
        top = np.sort(r64["qn"], 1)
        assert c.A < 2 or (top[:, -1] - top[:, -2]).min() > 1e-4, (top[:, -1] - top[:, -2]).min()
        # double DQN bootstraps from a smaller target value than plain DQN on some bootstrapping rows: the online and
        # target nets' argmax over Q(s') differ there
        boot = ~d["d"][i]
        at_online = r64["qt"][np.arange(c.B), np.argmax(r64["qn"], 1)]
        assert (at_online < r64["qt"].max(1))[boot].any()


def _set_fuse(lib, on):
    lib.xtb_set_fuse_heads(1 if on else 0)


@pytest.mark.parametrize("c", LEARNER, ids=[c.id for c in LEARNER])
def test_learner_step_against_float64(xb, tc_mode, c):
    """LR 0: the weights come back bitwise, and the loss, td_abs (max-norm), every parameter gradient (relative L2) and
    the global norm the optimiser computed are at most 4x torch-CPU fp32's distance from float64, + a floor of 6e-5
    (tensor cores) or 1e-5 (fp32) x max(1, sqrt(B / 128)), + the suite's ReLU flip allowance on the ReLU trunk's
    gradients, and a twentieth of it on the global norm, which those gradients dominate (observed on an H100 80GB HBM3
    at 700 W: the DqnCnn trunk at B = 512 on the tensor cores 2.3e-3, its norm 1.4e-4).  The reported norm is also the
    float64 norm of the device's own gradient within 1e-5, so a parameter the optimiser leaves out shows at every case.
    heads_plan() names the path the case is for."""
    lib = xb["lib"]
    _set_fuse(lib, c.fuse)
    try:
        lrn = _Learner(c)
        assert lrn.model.heads_plan() == c.plan, (lrn.model.heads_plan(), c.plan)
        ref = _learner_reference(c, lrn)
        w0 = lrn.net.get_weights()
        for k in w0:
            assert np.array_equal(w0[k], ref["w"][k]), k
        _assert_learner_regimes(c, ref)
        loss, td = lrn.step(_on_device(ref["d"]))
    finally:
        _set_fuse(lib, True)
    g = lrn.grads()
    gn = lrn.opt.grad_norm()
    w1 = lrn.net.get_weights()
    for k in w0:
        assert np.array_equal(w1[k], w0[k]), k
    r64, r32 = ref["f64"], ref["f32"]
    floor = (6e-5 if tc_mode == 1 else 1e-5) * max(1.0, np.sqrt(c.B / 128.0))
    flip = RELU_FLIP_TC if tc_mode == 1 else RELU_FLIP_F32
    heads = _heads(c)
    errs = {k: (l2_rel(g[k], r64["g"][k]), l2_rel(r32["g"][k], r64["g"][k])) for k in r64["g"]}
    errs["loss"] = (abs(loss - r64["loss"]) / max(1.0, abs(r64["loss"])), abs(r32["loss"] - r64["loss"]) / max(1.0, abs(r64["loss"])))
    errs["td_abs"] = (rel_err(td, r64["td"]), rel_err(r32["td"], r64["td"]))
    errs["grad_norm"] = (abs(gn - r64["norm"]) / r64["norm"], abs(r32["norm"] - r64["norm"]) / r64["norm"])
    record("dqn_step_vs_f64/%s/%s" % (c.id, "tcgen05" if tc_mode else "fp32"),
           {k: ["%.2e" % a, "%.2e" % b] for k, (a, b) in errs.items()})
    allow = {k: flip for k in r64["g"] if k not in heads}
    allow["grad_norm"] = flip / 20
    bad = {k: e for k, e in errs.items() if not e[0] <= 4 * e[1] + floor + allow.get(k, 0.0)}
    assert not bad, bad
    own = np.sqrt(sum(float((v.astype(np.float64) ** 2).sum()) for v in g.values()))
    assert abs(gn - own) <= 1e-5 * own, (gn, own)


def test_cases_cover_every_dueling_instantiation(xb):
    """probe the library over hidden widths and action counts: every heads_kernel<DuelingTdLoss> entry it can pick is
    named by some learner case, and the cases' plans are entries the probe found"""
    from xingtian_b200.model.dqn import DqnMlp
    seen = set()
    for hidden in (32, 64, 96, 128, 256, 288, 512, 544):
        for A in (1, 2, 4, 5, 8, 9):
            m = DqnMlp({"state_dim": [8], "action_dim": A, "max_batch": 8,
                        "model_config": {"dueling": True, "init_seed": 1, "HIDDEN_SIZE": hidden}})
            p = m.heads_plan()
            if p != (0, 0):
                seen.add(p)
                assert hidden // 32 <= p[0] and A <= p[1], (hidden, A, p)
            else:
                assert hidden > 512 or A > 8 or (hidden > 256 and A > 4), (hidden, A)
    assert seen == {(2, 8), (8, 4), (8, 8), (16, 4)}, seen
    covered = {c.plan for c in LEARNER if c.plan != (0, 0)}
    assert covered == seen, (covered, seen)
    assert any(c.plan == (0, 0) and c.dueling and c.fuse for c in LEARNER)


# ---- c. eager, graph capture, graph replay and the data-parallel path -----------------------------------------------
FORMS = [_L("cnn", 4, 64, dueling=True, plan=(8, 4)), _L("cnn", 4, 64)]
FORMS_BOUND = 4e-6     # reordered fp32 sums, relative L2 per tensor (observed <= 2.3e-7 on an H100 80GB HBM3 at 700 W)


@pytest.mark.parametrize("c", FORMS, ids=[c.id for c in FORMS])
def test_learner_step_forms_agree(xb, tc_mode, c):
    """eager, eager again, the graph call that captures, a replay and eager with a one-rank communicator installed (the
    gradient all-reduce runs) at LR 0, through the unweighted entry: the weights come back bitwise, the loss within 1e-6
    (bitwise when the fused heads' ordered reduction sums it), the gradients of the layers on the tensor cores and, on
    both kernel paths, those the fused heads' ordered reduction writes bitwise (the forward below the heads adds no
    partial sums with atomics, so their input is the same bits every call), every other gradient tensor within
    FORMS_BOUND of the first eager call's (relative L2; split-K weight-gradient partial sums and bias sums are added with
    atomics)"""
    lib = xb["lib"]
    lrn = _Learner(c)
    assert lrn.model.heads_plan() == c.plan
    w0 = lrn.net.get_weights()
    dd = _on_device(_learner_data(c))
    out = {}
    lrn.model.use_graph = False
    out["eager"] = (lrn.step(dd, plain=True)[0], lrn.grads())
    out["eager_again"] = (lrn.step(dd, plain=True)[0], lrn.grads())
    lrn.model.use_graph = True
    c0, r0 = lib.xtb_graph_capture_count(), lib.xtb_graph_replay_count()
    out["capture"] = (lrn.step(dd, plain=True)[0], lrn.grads())
    assert (lib.xtb_graph_capture_count() - c0, lib.xtb_graph_replay_count() - r0) == (1, 1)
    out["replay"] = (lrn.step(dd, plain=True)[0], lrn.grads())
    assert (lib.xtb_graph_capture_count() - c0, lib.xtb_graph_replay_count() - r0) == (1, 2)
    lrn.model.use_graph = False
    with one_rank_comm():
        out["one_rank_comm"] = (lrn.step(dd, plain=True)[0], lrn.grads())
    w1 = lrn.net.get_weights()
    for k in w0:
        assert np.array_equal(w1[k], w0[k]), k
    le, ge = out["eager"]
    on_tc = [n for i, (n, _, _, _) in enumerate(lrn.net.arch["layers"]) if tc_mode == 1 and lrn.net.layer_plan(i)["tc"]]
    exact = {n + sfx for n in on_tc for sfx in ("/kernel", "/bias")}
    if c.plan[0]:
        exact |= _heads(c)
    assert exact or tc_mode == 0
    errs = {form: {k: l2_rel(g[k], ge[k]) for k in ge} for form, (_, g) in out.items()}
    record("dqn_step_forms/%s/%s" % (c.id, "tcgen05" if tc_mode else "fp32"),
           {"loss": {form: "%.9g" % l for form, (l, _) in out.items()}, "bitwise": sorted(exact),
            "grad_l2_rel_to_eager": {form: {k: "%.1e" % e for k, e in es.items() if e > 0} for form, es in errs.items()}})
    for form, (l, g) in out.items():
        assert (l == le) if c.plan[0] else abs(l - le) <= 1e-6 * abs(le), (form, l, le)
        bad = {k: e for k, e in errs[form].items() if not (e == 0.0 if k in exact else e <= FORMS_BOUND)}
        assert not bad, (form, bad)


# ---- d. the clip and Adam wiring ------------------------------------------------------------------------------------
B1, B2 = 1.0 - _f32(0.9), 1.0 - _f32(0.999)


@pytest.mark.parametrize("kind", ["cnn", "mlp"])
def test_learner_step_clips_per_tensor_and_takes_one_adam_step(xb, tc_mode, kind):
    """One step at LR 1.5e-4 with rewards N(0, 30^2).  DqnCnn clips each tensor to norm 10 (Keras clipnorm); some of its
    tensors' norms exceed 10 and some do not.  DqnMlp does not clip.
    - The norm the optimiser computed is the float64 norm of the device's own gradient within 1e-5.
    - After the first step Adam's moments are (1 - beta1) g' and (1 - beta2) g'^2 of the per-tensor clipped gradient g'
      in float64, within 1e-6 relative L2 per tensor.
    - The update is one TFAdam step (eps 1e-7) of g' in float64, within 1e-5 relative L2."""
    c = _L("cnn", 4, 64) if kind == "cnn" else _L("mlp", 4, 64, dueling=True, hidden=128, plan=(8, 4))
    lr = 1.5e-4
    lrn = _Learner(c, lr=lr)
    w0 = lrn.net.get_weights()
    lrn.step(_on_device(_learner_data(c, rewards=30.0)))
    g = lrn.grads()
    gn = lrn.opt.grad_norm()
    w1 = lrn.net.get_weights()
    names = list(w0)
    with orc.precision("f64"):
        gl = [torch.from_numpy(g[k].astype(np.float64)) for k in names]
        n64 = float(np.sqrt(sum(float((t ** 2).sum()) for t in gl)))
        norms = [float(t.norm()) for t in gl]
        clipped = orc.clip_per_tensor(gl, 10.0) if kind == "cnn" else gl
        params = [torch.from_numpy(w0[k].astype(np.float64)) for k in names]
        orc.TFAdam(params, lr, eps=1e-7).step(clipped)
    upd = np.concatenate([(w1[k].astype(np.float64) - w0[k]).ravel() for k in names])
    want = np.concatenate([(p.numpy().astype(np.float32).astype(np.float64) - w0[k]).ravel() for k, p in zip(names, params)])
    err = l2_rel(upd, want)
    mom, var = lrn.net.get_weights(lrn.opt.m), lrn.net.get_weights(lrn.opt.v)
    m_err = max(l2_rel(mom[k], B1 * t.numpy()) for k, t in zip(names, clipped))
    v_err = max(l2_rel(var[k], B2 * t.numpy() ** 2) for k, t in zip(names, clipped))
    record("dqn_step_clip_adam/%s/%s" % (kind, "tcgen05" if tc_mode else "fp32"),
           {"grad_norm": "%.6g" % gn, "tensor_norms": ["%.3g" % n for n in norms], "norm_rel_err": "%.2e" % (abs(gn - n64) / n64),
            "m_l2_rel": "%.2e" % m_err, "v_l2_rel": "%.2e" % v_err, "update_l2_rel": "%.2e" % err})
    if kind == "cnn":
        assert max(norms) > 10.0 and min(norms) < 10.0, norms
    assert abs(gn - n64) <= 1e-5 * n64, (gn, n64)
    assert m_err <= 1e-6 and v_err <= 1e-6, (m_err, v_err)
    assert err <= 1e-5, err
