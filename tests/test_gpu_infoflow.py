"""GPU tier: DqnInfoFlowModel's device step and predict against the float64 restatement (tests/infoflow_oracle.py), and a
CPU check that the InfoFlow kernels and the generalised GRU kernels compile for sm_90a without spills.

Bounds: the same restatement run in fp32 measures what fp32 rounding alone does to each quantity; the device result must
stay within 8x that distance of the float64 result, plus 1e-5 of the quantity's magnitude.  On the tensor cores the
floor for the weights and the Adam slots is 1e-4, as in the QMIX test: the head's weight gradients are reduced over the
rows from bf16 hi / lo operand planes, and Adam divides each gradient by its own root mean square, so a gradient near
zero turns its small absolute error into an update of the order of the learning rate.  hard_sigmoid has kinks at +-2.5,
so every case asserts that the float64 run's gate pre-activations stay at least 1e-4 away from them."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
import infoflow_oracle as io

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
VOCAB = 40
GAMMA = 0.9


def session(item_dim, emb_dim, user_dim, B, n_steps, seed, counts=None, done=None):
    """Seeded embedding table, weights and n_steps packed minibatches (DQNInfoFlowAlg.pack's form)."""
    rng = np.random.default_rng(seed)
    U = item_dim * emb_dim
    table = (rng.standard_normal((VOCAB, emb_dim)) * 0.5).astype(np.float32)
    D = user_dim * emb_dim + 3 * U
    w = {}
    for s in ("gru", "gru_1"):
        w[s + "/kernel"] = rng.uniform(-1, 1, (U, 3 * U)) * np.sqrt(6.0 / (4 * U))
        w[s + "/recurrent_kernel"] = rng.uniform(-1, 1, (U, 3 * U)) * np.sqrt(3.0 / U)
        w[s + "/bias"] = rng.uniform(-0.1, 0.1, 3 * U)
    for name, (k, n) in (("dense", (D, 128)), ("dense_1", (128, 128)), ("q_value", (128, 1))):
        w[name + "/kernel"] = rng.uniform(-1, 1, (k, n)) * np.sqrt(6.0 / (k + n))
        w[name + "/bias"] = rng.uniform(-0.1, 0.1, n)
    w = {k: v.astype(np.float32) for k, v in w.items()}
    batches = []
    for _ in range(n_steps):
        cnt = rng.integers(1, 12, B) if counts is None else np.asarray(counts)
        dn = rng.random(B) < 0.3 if done is None else np.full(B, done)
        ids = lambda *s: rng.integers(0, VOCAB, s).astype(np.int32)
        b = dict(user=ids(B, user_dim), click=ids(B, 5 * item_dim), noclick=ids(B, 5 * item_dim), item=ids(B, item_dim),
                 next_user=ids(B, user_dim), next_click=ids(B, 5 * item_dim), next_noclick=ids(B, 5 * item_dim),
                 cand_off=np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32), cand_item=ids(int(cnt.sum()), item_dim),
                 reward=rng.uniform(-1, 1, B), done=dn.astype(np.int32))
        batches.append(b)
    return table, w, batches


def oracle_run(table, w, batches, last_act, prec, pre=None):
    with orc.precision(prec):
        lrn = io.InfoflowLearner(w, table, last_act, GAMMA)
        out = [lrn.step(b, pre=pre) for b in batches]
        return np.array([o[0] for o in out]), [o[1] for o in out], lrn.weights(), lrn.slots()


def margins_ok(table, w, batches, last_act):
    pre = []
    oracle_run(table, w, batches, last_act, "f64", pre)
    m = min(float(torch.min(torch.abs(torch.abs(p) - 2.5))) for p in pre)
    assert m >= 1e-4, "a gate pre-activation lies {:.3g} from a hard_sigmoid kink: pick another seed".format(m)


def close(dev, f64, f32, what, floor=1e-5):
    dev, f64, f32 = (np.asarray(x, np.float64) for x in (dev, f64, f32))
    bound = 8 * np.abs(f32 - f64) + floor * max(1.0, float(np.abs(f64).max()))
    err = np.abs(dev - f64)
    assert np.all(err <= bound), "{}: max error {:.3g} (bound there {:.3g})".format(what, err.max(), bound.flat[np.argmax(err - bound)])


@pytest.fixture(scope="module")
def tmpdir_mod():
    with tempfile.TemporaryDirectory() as d:
        yield d


def make(table, item_dim, emb_dim, user_dim, last_act="linear", use_graph=True, d=None):
    from xingtian_b200.model.dqn_infoflow import DqnInfoFlowModel
    path = os.path.join(d or tempfile.mkdtemp(), "emb_%d_%d.csv" % (VOCAB, emb_dim))
    np.savetxt(path, table.astype(np.float64), delimiter=",", fmt="%.9g")
    info = dict(state_dim=[1], action_dim=1, vocab_size=VOCAB, emb_dim=emb_dim, user_dim=user_dim, item_dim=item_dim,
                input_type="int32", embeddings=path, last_activate=last_act, model_config=dict(init_seed=0, use_cuda_graph=use_graph))
    return DqnInfoFlowModel(info)


def set_all(m, w):
    m.set_weights({k: v for k, v in w.items()})


def check_train(m, table, w, batches, last_act, floor=1e-5):
    set_all(m, w)
    m.set_gamma(GAMMA)
    losses = [m._train_packed(b) for b in batches]
    l64, t64, w64, s64 = oracle_run(table, w, batches, last_act, "f64")
    l32, t32, w32, s32 = oracle_run(table, w, batches, last_act, "f32")
    close(losses, l64, l32, "loss")
    dev = m.variables()
    for k in io.TRAINABLE:
        close(dev[k], w64[k], w32[k], k, floor)
    mdev, vdev = m.opt.m.cpu().numpy(), m.opt.v.cpu().numpy()
    for i, k in enumerate(io.TRAINABLE):
        off, shape = m.vars[k]
        sl = slice(off, off + int(np.prod(shape)))
        close(mdev[sl], s64[0][i].reshape(-1), s32[0][i].reshape(-1), k + " m", floor)
        close(vdev[sl], s64[1][i].reshape(-1), s32[1][i].reshape(-1), k + " v", floor)


@pytest.fixture(params=[1, 0], ids=["tc", "fp32"])
def tc_mode(request):
    from xingtian_b200 import capi
    lib = capi.lib()
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(request.param)
    yield request.param
    lib.xtb_set_tc_mode(old)


CASES = [  # item_dim, emb_dim, user_dim, B, last_act, steps, seed
    (1, 8, 1, 32, "linear", 3, 1),
    (3, 8, 4, 1, "sigmoid", 3, 2),
    (3, 32, 4, 256, "relu", 2, 3),
    (1, 128, 1, 32, "linear", 2, 4),
    (1, 137, 4, 32, "sigmoid", 2, 5),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: "id{}-E{}-u{}-B{}-{}".format(*c[:5]))
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])
def test_train_matches_oracle(case, use_graph, tc_mode, tmpdir_mod):
    item_dim, E, ud, B, act, steps, seed = case
    table, w, batches = session(item_dim, E, ud, B, steps, seed)
    margins_ok(table, w, batches, act)
    m = make(table, item_dim, E, ud, act, use_graph, tmpdir_mod)
    check_train(m, table, w, batches, act, 1e-4 if tc_mode else 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("done", [True, False], ids=["all_done", "none_done"])
def test_all_done_and_none_done(done, tc_mode, tmpdir_mod):
    table, w, batches = session(3, 8, 4, 32, 2, 6, done=done)
    margins_ok(table, w, batches, "linear")
    check_train(make(table, 3, 8, 4, "linear", True, tmpdir_mod), table, w, batches, "linear", 1e-4 if tc_mode else 1e-5)


@pytest.mark.gpu
def test_predict_and_targets_match_oracle_exactly_on_device_q(tmpdir_mod):
    table, w, batches = session(3, 8, 4, 32, 1, 7)
    m = make(table, 3, 8, 4, "linear", True, tmpdir_mod)
    set_all(m, w)
    m.set_gamma(GAMMA)
    b = batches[0]
    n = np.diff(b["cand_off"])
    rep = lambda a: np.repeat(a, n, axis=0)
    state = dict(user_input=rep(b["next_user"]), history_click=rep(b["next_click"]), history_no_click=rep(b["next_noclick"]),
                 item_input=b["cand_item"])
    q = m.predict(state)
    assert q.dtype == np.float32 and q.shape == (int(n.sum()),)
    with orc.precision("f64"):
        q64 = io.InfoflowLearner(w, table, "linear", GAMMA).predict(*[state[k] for k in ("user_input", "history_click",
                                                                                           "history_no_click", "item_input")])
    with orc.precision("f32"):
        q32 = io.InfoflowLearner(w, table, "linear", GAMMA).predict(*[state[k] for k in ("user_input", "history_click",
                                                                                           "history_no_click", "item_input")])
    close(q, q64, q32, "predict")
    tgt = torch.zeros(32, dtype=torch.float32, device="cuda")
    m._train_packed(b, target_out=tgt)
    want = io.td_targets(q, b["cand_off"], b["reward"], b["done"], GAMMA).astype(np.float32)
    np.testing.assert_array_equal(tgt.cpu().numpy(), want)


@pytest.mark.gpu
def test_nan_candidate_propagates_to_the_target(tmpdir_mod):
    table, w, batches = session(1, 8, 1, 4, 1, 8, done=False)
    w["q_value/bias"] = np.array([np.nan], np.float32)
    m = make(table, 1, 8, 1, "linear", True, tmpdir_mod)
    set_all(m, w)
    m.set_gamma(GAMMA)
    tgt = torch.zeros(4, dtype=torch.float32, device="cuda")
    m._train_packed(batches[0], target_out=tgt)
    assert np.all(np.isnan(tgt.cpu().numpy()))


@pytest.mark.gpu
def test_same_bucket_causes_no_new_capture(tmpdir_mod):
    from xingtian_b200 import capi
    lib = capi.lib()
    table, w, batches = session(1, 8, 1, 8, 3, 9, counts=[5] * 8)
    batches[1]["cand_off"] = np.concatenate([[0], np.cumsum([6] * 8)]).astype(np.int32)      # 48 rows: same 64 bucket
    batches[1]["cand_item"] = np.random.default_rng(0).integers(0, VOCAB, (48, 1)).astype(np.int32)
    batches[2]["cand_off"] = np.concatenate([[0], np.cumsum([9] * 8)]).astype(np.int32)      # 72 rows: the 128 bucket
    batches[2]["cand_item"] = np.random.default_rng(1).integers(0, VOCAB, (72, 1)).astype(np.int32)
    m = make(table, 1, 8, 1, "linear", True, tmpdir_mod)
    set_all(m, w)
    m.set_gamma(GAMMA)
    m._train_packed(batches[0])
    c0 = lib.xtb_graph_capture_count()
    m._train_packed(batches[1])
    assert lib.xtb_graph_capture_count() == c0
    m._train_packed(batches[2])
    assert lib.xtb_graph_capture_count() == c0 + 1


@pytest.mark.gpu
def test_weights_round_trip_and_npz(tmpdir_mod):
    table, w, batches = session(3, 8, 4, 32, 1, 10)
    m = make(table, 3, 8, 4, "relu", True, tmpdir_mod)
    m.set_gamma(GAMMA)
    m._train_packed(batches[0])
    lst = m.get_weights()
    assert len(lst) == 13 and lst[-1].shape == (VOCAB, 8)
    m2 = make(table * 2, 3, 8, 4, "relu", True, tmpdir_mod)
    m2.set_weights(lst)
    for a, b in zip(m2.get_weights(), lst):
        np.testing.assert_array_equal(a, b)
    path = m.save_model(os.path.join(tmpdir_mod, "actor_00001"))
    m3 = make(table * 3, 3, 8, 4, "relu", True, tmpdir_mod)
    m3.load_model(path)
    for a, b in zip(m3.get_weights(), lst):
        np.testing.assert_array_equal(a, b)
    with np.load(path) as f:
        assert sorted(f.files) == sorted(io.TRAINABLE + ["Emb/embeddings"])
    bad = list(lst)
    bad[0] = bad[0][:, :-1]
    with pytest.raises(ValueError):
        m2.set_weights(bad)
    with pytest.raises(KeyError):
        m2.set_weights({"nope": lst[0]})


@pytest.mark.gpu
def test_algorithm_trains_and_syncs_target(tmpdir_mod):
    from xingtian_b200.algorithm.dqn_infoflow import DQNInfoFlowAlg
    rng = np.random.default_rng(11)
    table = (rng.standard_normal((VOCAB, 4)) * 0.5).astype(np.float32)
    path = os.path.join(tmpdir_mod, "alg_emb.csv")
    np.savetxt(path, table, delimiter=",")
    info = dict(actor=dict(model_name="DqnInfoFlowModel", state_dim=[1], action_dim=1, vocab_size=VOCAB, emb_dim=4, user_dim=2,
                           item_dim=2, input_type="int32", embeddings=path, last_activate="linear", model_config=dict(init_seed=0)))
    alg = DQNInfoFlowAlg(info, dict(instance_num=1, agent_num=1, batch_size=4, item_dim=2, user_dim=2, target_update_freq=2,
                                    gamma=0.99))
    st = lambda: dict(user=rng.integers(0, VOCAB, 2), clicked_items=rng.integers(0, VOCAB, 10), viewed_items=rng.integers(0, VOCAB, 10),
                      candidate_items=rng.integers(0, VOCAB, (int(rng.integers(1, 5)), 2)))
    data = dict(cur_state=[st() for _ in range(6)], action=[rng.integers(0, VOCAB, 2) for _ in range(6)], reward=[0.5] * 6,
                next_state=[st() for _ in range(6)], done=[False, True] * 3)
    alg.prepare_data(data)
    loss = alg.train(episode_num=1)
    assert np.isfinite(loss)
    assert not all(np.array_equal(a, b) for a, b in zip(alg.actor.get_weights(), alg.target_actor.get_weights()))
    alg.train(episode_num=2)
    for a, b in zip(alg.actor.get_weights(), alg.target_actor.get_weights()):
        np.testing.assert_array_equal(a, b)


@pytest.mark.gpu
def test_rejections(tmpdir_mod):
    from xingtian_b200 import capi
    table, w, batches = session(1, 8, 1, 4, 1, 12)
    with pytest.raises(ValueError):
        make(np.zeros((VOCAB, 138), np.float32), 1, 138, 1, "linear", True, tmpdir_mod)
    d = capi.InfoflowDesc()
    d.user_dim, d.item_dim, d.emb_dim, d.vocab, d.batch, d.last_act, d.gamma = 1, 1, 138, VOCAB, 4, 0, 0.9
    gn = 6 * 138 * 138 + 3 * 138
    d.gru_off, d.gru1_off, d.head_off = 0, (gn + 63) // 64 * 64, 2 * ((gn + 63) // 64 * 64)
    d.table = torch.zeros(VOCAB * 138, device="cuda").data_ptr()
    h = C.c_void_p()
    assert capi.lib().xtb_infoflow_create(C.byref(d), C.byref(h)) == -1
    d.emb_dim = 137
    gn = 6 * 137 * 137 + 3 * 137
    d.gru1_off, d.head_off = (gn + 63) // 64 * 64, 2 * ((gn + 63) // 64 * 64)
    assert capi.lib().xtb_infoflow_create(C.byref(d), C.byref(h)) == 0
    capi.lib().xtb_infoflow_destroy(h)
    with pytest.raises(KeyError):
        make(table, 1, 8, 1, "hard_sigmoid", True, tmpdir_mod)


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which(NVCC)), reason="nvcc not available")
def test_infoflow_and_gru_kernels_do_not_spill(repo_root, tmp_path):
    csrc = os.path.join(repo_root, "xingtian_b200", "csrc")
    src = tmp_path / "infoflow_only.cu"
    src.write_text('#include "{0}/gemm_f32.cuh"\n#include "{0}/qmix.cuh"\n#include "{0}/infoflow.cuh"\n'.format(csrc))
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o",
           str(tmp_path / "k.cubin"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    kernels, cur = {}, None
    for line in (res.stdout + res.stderr).splitlines():
        mt = re.search(r"Compiling entry function '([^']+)'", line)
        if mt:
            cur = mt.group(1) if ("infoflow" in mt.group(1) or "gru" in mt.group(1)) else None
            continue
        mt = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and mt:
            kernels[cur] = tuple(int(x) for x in mt.groups())
    assert len(kernels) == 6, sorted(kernels)
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
