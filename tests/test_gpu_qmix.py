"""GPU tier: QMixModel's device training step and one-step inference against the float64 restatement
(tests/qmix_oracle.py).

Bounds: the same restatement run in fp32 (orc.precision("f32")) measures what fp32 rounding alone does to each quantity;
the device result must stay within 8x that distance of the float64 result, plus 1e-5 of the quantity's magnitude (the
tensor-core layers carry each fp32 operand as two bf16 planes, which is fp32-like but not identical rounding)."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
import qmix_oracle as qo

pytestmark = pytest.mark.gpu

OBS, SD, H, A, E, HE = 6, 7, 32, 5, 8, 16


def make(n, double_q=True, L=8, B=4, seed=0, use_graph=True, H=H, **over):
    from xingtian_b200.model.qmix import QMixModel
    mc = dict(gamma=0.99, lr=0.0005, grad_norm_clip=10, n_agents=n, obs_shape=OBS, rnn_hidden_dim=H, episode_limit=L, n_actions=A,
              batch_size=B, state_shape=[SD], mixing_embed_dim=E, hypernet_embed=HE, hypernet_layers=2, use_double_q=double_q,
              init_seed=seed, use_cuda_graph=use_graph)
    mc.update(over)
    return QMixModel(dict(model_config=mc, scene="train"))


def oracle_run(eval_w, target_w, batches, prec, double_q):
    with orc.precision(prec):
        lrn = qo.QmixLearner(eval_w, target_w, 0.0005, 10, 0.99, double_q)
        losses = [lrn.step(b) for b in batches]
        w = {k: v.detach().numpy().astype(np.float64) for k, v in lrn.w.items()}
        return np.array(losses), w, lrn.slots()


def close(dev, f64, f32, what):
    dev, f64, f32 = (np.asarray(x, np.float64) for x in (dev, f64, f32))
    bound = 8 * np.abs(f32 - f64) + 1e-5 * max(1.0, float(np.abs(f64).max()))
    err = np.abs(dev - f64)
    assert np.all(err <= bound), "{}: max error {:.3g} (bound there {:.3g})".format(what, err.max(), bound.flat[np.argmax(err - bound)])


# (n_agents, double Q, full length, batch, rnn_hidden_dim, episode_limit).  B n > 132 sequences puts two sequences in a
# GRU CTA (qmix.yaml's batch 32 and hidden 64 with 5 agents); hidden 128 is the largest the GRU kernels take.
CASES = [(1, True, False, 4, H, 8), (2, True, True, 4, H, 8), (2, False, False, 4, H, 8), (5, True, False, 4, H, 8),
         (5, False, True, 4, H, 8), (5, True, False, 32, 64, 4), (2, True, True, 4, 128, 4)]


@pytest.mark.parametrize("n,double_q,full,B,hidden,L", CASES)
@pytest.mark.parametrize("steps", [1, 3])
def test_train_matches_oracle(n, double_q, full, B, hidden, L, steps):
    torch.cuda.set_device(0)
    m = make(n, double_q, L=L, B=B, H=hidden)
    w0, t0 = m.variables(m.params), m.variables(m.target)
    batches = [qo.synth_batch(10 * s + n, B, L, n, A, OBS, SD, max_ep_t=(L + 1 if full else min(L, 3 + s))) for s in range(steps)]
    dev_losses = [m.train(*qo.model_args(b)) for b in batches]
    l64, w64, s64 = oracle_run(w0, t0, batches, "f64", double_q)
    l32, w32, s32 = oracle_run(w0, t0, batches, "f32", double_q)
    close(dev_losses, l64, l32, "loss")
    wd = m.variables(m.params)
    ms, mg = m.variables(m.opt.m), m.variables(m.opt.mean_grad)
    for k in w64:
        close(wd[k], w64[k], w32[k], k)
        close(ms[k], s64[k][0], s32[k][0], k + " ms")
        close(mg[k], s64[k][1], s32[k][1], k + " mg")


def test_graph_replay_across_lengths_matches_eager():
    """One captured graph replayed for three max_ep_t values against eager launches of the same step.  The first loss
    is computed before any update and must be identical; after an update the engine's split-K dense weight gradients
    (atomic adds, not ordered) may round differently, so later steps are compared to fp32 rounding."""
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    L, B, n = 8, 4, 2
    g, e = make(n, use_graph=True), make(n, use_graph=False)
    replays = capi.lib().xtb_graph_replay_count()
    for s, t in enumerate((3, L + 1, 6)):
        b = qo.synth_batch(s, B, L, n, A, OBS, SD, max_ep_t=t)
        lg, le = g.train(*qo.model_args(b)), e.train(*qo.model_args(b))
        if s == 0:
            assert lg == le
        else:
            assert abs(lg - le) <= 1e-5 * max(1.0, abs(le)), (s, lg, le)
    assert capi.lib().xtb_graph_replay_count() - replays == 3
    for a, c in ((g.params, e.params), (g.opt.m, e.opt.m), (g.opt.mean_grad, e.opt.mean_grad)):
        torch.testing.assert_close(a, c, rtol=1e-5, atol=1e-7)


def test_new_kernels_reductions_are_bitwise_reproducible():
    """The loss, the mixer's gradients and the GRU's weight gradients (the reductions of the QMIX kernels and their
    GEMMs) repeat bit for bit; the engine's split-K weight gradients of the dense layers are not part of this."""
    torch.cuda.set_device(0)
    out = []
    for _ in range(2):
        m = make(5, seed=3)
        b = qo.synth_batch(7, 4, 8, 5, A, OBS, SD, max_ep_t=7)
        loss = m.train(*qo.model_args(b))
        g = m.variables(m.grads, mixer=False)
        out.append((loss, [g[k] for k in (qo.GATES_K, qo.GATES_B, qo.CAND_K, qo.CAND_B)],
                    [m.fc2.tensor_grad("dense_1").clone()] + [m.hyper.tensor_grad(h).clone() for h in
                                                             ("hyper_w1/dense_1", "hyper_b1/dense", "hyper_w_final/dense_1",
                                                              "val_for_bias/dense_1")]))
    assert out[0][0] == out[1][0]
    assert all(np.array_equal(a, c) for a, c in zip(out[0][1], out[1][1]))
    assert all(torch.equal(a, c) for a, c in zip(out[0][2], out[1][2]))


def test_infer_actions_carries_the_hidden_state():
    torch.cuda.set_device(0)
    n = 3
    m = make(n)
    b = qo.synth_batch(1, 4, 8, n, A, OBS, SD, max_ep_t=9)
    m.train(*qo.model_args(b))
    m.assign_explore_agent()
    w = m.variables(m.explore, mixer=False)
    rng = np.random.default_rng(5)
    for episode in range(2):
        m.reset_hidden_state()
        h64 = h32 = None
        for step in range(4):
            x = rng.normal(size=(1, 1, n, OBS)).astype(np.float32)
            q = m.infer_actions(x)
            assert q.shape == (1, n, A)
            ref = {}
            for prec in ("f64", "f32"):
                with orc.precision(prec):
                    wt = {k: qo._t(v) for k, v in w.items()}
                    h0 = h64 if prec == "f64" else h32
                    qr, hT = qo.agent_forward(wt, qo._t(x), [1] * n, h0)
                    ref[prec] = qr.numpy().reshape(1, n, A)
                    if prec == "f64":
                        h64 = hT
                    else:
                        h32 = hT
            close(q, ref["f64"], ref["f32"], "q episode %d step %d" % (episode, step))


def test_weights_round_trip():
    torch.cuda.set_device(0)
    m = make(2)
    w = m.get_weights()
    names = ["explore_agent/" + s for s in ("dense/kernel", "dense/bias", qo.GATES_K, qo.GATES_B, qo.CAND_K, qo.CAND_B,
                                            "dense_1/kernel", "dense_1/bias")]
    assert list(w) == names
    assert w["explore_agent/" + qo.GATES_K].shape == (2 * H, 2 * H) and w["explore_agent/" + qo.CAND_K].shape == (2 * H, H)
    assert np.all(w["explore_agent/" + qo.GATES_B] == 1.0) and np.all(w["explore_agent/" + qo.CAND_B] == 0.0)
    m.assign_explore_agent()
    ev = m.variables(m.params, mixer=False)
    assert all(np.array_equal(m.get_weights()["explore_agent/" + k], v) for k, v in ev.items())
    m.set_weights(w)
    assert all(np.array_equal(m.get_weights()[k], v) for k, v in w.items())
    with tempfile.TemporaryDirectory() as d:
        path = m.save_explore_agent_weights(os.path.join(d, "actor00001"))
        m2 = make(2, seed=9)
        m2.restore_explorer_variable(os.path.join(d, "actor00001"))
        assert all(np.array_equal(m2.get_weights()[k], v) for k, v in w.items())
        assert path.endswith(".npz")
    with pytest.raises(KeyError):
        m.set_weights({"nothing": np.zeros(1)})
    b = qo.synth_batch(2, 4, 8, 2, A, OBS, SD, max_ep_t=9)
    m.train(*qo.model_args(b))
    assert not all(np.array_equal(a, c) for a, c in zip(m.variables(m.params).values(), m.variables(m.target).values()))
    m.assign_targets()
    assert all(np.array_equal(a, c) for a, c in zip(m.variables(m.params).values(), m.variables(m.target).values()))


def test_rejected_arguments_launch_nothing():
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    import ctypes as C
    lib = capi.lib()
    for over in (dict(n_actions=256), dict(rnn_hidden_dim=160), dict(n_agents=33), dict(mixing_embed_dim=129)):
        with pytest.raises(RuntimeError):
            make(2, **over)
    m = make(2)
    before = lib.xtb_launch_count()
    desc = capi.QmixDesc()
    desc.batch, desc.episode_limit, desc.n_agents, desc.gamma, desc.gru_off = 4, 8, 33, 0.99, m.gru_off
    h = C.c_void_p()
    assert lib.xtb_qmix_create(m.fc1.handle, m.fc2.handle, m.hyper.handle, C.byref(desc), C.byref(h)) == -1
    desc.n_agents, desc.gru_off = 2, 0
    assert lib.xtb_qmix_create(m.fc1.handle, m.fc2.handle, m.hyper.handle, C.byref(desc), C.byref(h)) == -1
    b = qo.synth_batch(0, 4, 8, 2, A, OBS, SD, max_ep_t=9)
    bad_len = dict(b, seq_len=np.full(8, 10, np.int32))
    with pytest.raises(ValueError):
        m.train(*qo.model_args(bad_len))
    bad_act = dict(b, actions=np.full_like(b["actions"], A))
    with pytest.raises(ValueError):
        m.train(*qo.model_args(bad_act))
    bt = capi.QmixBatch()
    assert lib.xtb_qmix_train(m.handle, m.opt.handle, C.c_void_p(m.target.data_ptr()), C.byref(bt), C.c_void_p(0), 0, None) == -1
    assert lib.xtb_launch_count() == before
