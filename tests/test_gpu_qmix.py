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


def make(n, double_q=True, L=8, B=4, seed=0, use_graph=True, H=H, E=E, HE=HE, A=A, obs=OBS, sd=SD, **over):
    from xingtian_b200.model.qmix import QMixModel
    mc = dict(gamma=0.99, lr=0.0005, grad_norm_clip=10, n_agents=n, obs_shape=obs, rnn_hidden_dim=H, episode_limit=L, n_actions=A,
              batch_size=B, state_shape=[sd], mixing_embed_dim=E, hypernet_embed=HE, hypernet_layers=2, use_double_q=double_q,
              init_seed=seed, use_cuda_graph=use_graph)
    mc.update(over)
    return QMixModel(dict(model_config=mc, scene="train"))


@pytest.fixture(params=[1, 0], ids=["tc", "fp32"])
def tc_mode(request):
    from xingtian_b200 import capi
    lib = capi.lib()
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(request.param)
    yield request.param
    lib.xtb_set_tc_mode(old)


def params_changed(m):
    """After a host-side write into m.params: refresh the bf16 planes the tensor-core layers read."""
    for net in (m.fc1, m.fc2, m.hyper):
        net.params_changed()


def oracle_run(eval_w, target_w, batches, prec, double_q):
    with orc.precision(prec):
        lrn = qo.QmixLearner(eval_w, target_w, 0.0005, 10, 0.99, double_q)
        losses = [lrn.step(b) for b in batches]
        w = {k: v.detach().numpy().astype(np.float64) for k, v in lrn.w.items()}
        return np.array(losses), w, lrn.slots()


def close(dev, f64, f32, what, floor=1e-5):
    dev, f64, f32 = (np.asarray(x, np.float64) for x in (dev, f64, f32))
    bound = 8 * np.abs(f32 - f64) + floor * max(1.0, float(np.abs(f64).max()))
    err = np.abs(dev - f64)
    assert np.all(err <= bound), "{}: max error {:.3g} (bound there {:.3g})".format(what, err.max(), bound.flat[np.argmax(err - bound)])


def check_train(m, batches, double_q, floor=1e-5):
    """Train m on the batches and compare every loss, every variable and both RMSProp slots with the restatement started
    from m's weights (close() with the given magnitude floor); returns the float64 weights."""
    w0, t0 = m.variables(m.params), m.variables(m.target)
    dev_losses = [m.train(*qo.model_args(b)) for b in batches]
    l64, w64, s64 = oracle_run(w0, t0, batches, "f64", double_q)
    l32, w32, s32 = oracle_run(w0, t0, batches, "f32", double_q)
    close(dev_losses, l64, l32, "loss", floor)
    wd = m.variables(m.params)
    ms, mg = m.variables(m.opt.m), m.variables(m.opt.mean_grad)
    for k in w64:
        close(wd[k], w64[k], w32[k], k, floor)
        close(ms[k], s64[k][0], s32[k][0], k + " ms", floor)
        close(mg[k], s64[k][1], s32[k][1], k + " mg", floor)
    return w64


def gru_groups(B, n):
    """Sequences per GRU CTA that xtb_qmix_create picks for B n sequences at the test widths (up to 8, over 132 SMs)."""
    return max(1, min(8, -(-B * n // 132)))


# (n_agents, double Q, full length, batch, rnn_hidden_dim, episode_limit, mixing embed, hypernet embed, actions).
# - B n > 132 sequences puts several sequences in a GRU CTA: 160 gives G = 2 (qmix.yaml's batch 32 and hidden 64 with 5
#   agents), 135 G = 2 with one sequence in the last CTA, 1057 G = 8 (the most) with one sequence in the last CTA.
# - Hidden 137 is the widest GRU create accepts (3H^2 + 7H floats of shared memory at one sequence per CTA); 134
#   sequences would take G = 2, which does not fit, so create drops to G = 1.  Hidden 1, 17 and 33 are not multiples
#   of 32.
# - The mixer warp keeps agent a on lane a and embed unit j on lane j % 32, slot j / 32: E 128 fills all four slots and
#   32 agents all lanes; E 100 leaves slot 3 partly filled, E 33 puts one unit in slot 1, E 1 is the narrowest.
# - The target's argmax / max walks the actions lane, lane + 32, ...: 33, 40 and 255 actions reach the second and later
#   strides (255 is the most create accepts).
# A case's id leaves out the mixer and action widths when they are the defaults.
CASES = [(1, True, False, 4, H, 8, E, HE, A), (2, True, True, 4, H, 8, E, HE, A), (2, False, False, 4, H, 8, E, HE, A),
         (5, True, False, 4, H, 8, E, HE, A), (5, False, True, 4, H, 8, E, HE, A), (5, True, False, 32, 64, 4, E, HE, A),
         (2, True, True, 4, 128, 4, E, HE, A),
         (32, True, False, 2, H, 4, 128, 64, A), (32, False, True, 2, H, 4, 128, 64, A),
         (7, False, False, 4, H, 4, 100, HE, 40), (3, True, True, 4, H, 4, 33, HE, 33), (1, True, False, 4, H, 4, 1, HE, 255),
         (2, True, False, 4, 1, 4, E, HE, A), (2, False, True, 4, 17, 4, E, HE, A), (3, True, False, 4, 33, 4, E, HE, A),
         (2, True, True, 67, 137, 4, E, HE, A), (5, True, False, 27, H, 4, E, HE, A), (7, False, True, 151, H, 2, E, HE, A)]


def _case_id(c):
    return "-".join(str(x) for x in (c[:6] if c[6:] == (E, HE, A) else c))


@pytest.mark.parametrize("n,double_q,full,B,hidden,L,embed,hyper_embed,actions", CASES, ids=[_case_id(c) for c in CASES])
@pytest.mark.parametrize("steps", [1, 3])
def test_train_matches_oracle(n, double_q, full, B, hidden, L, embed, hyper_embed, actions, steps):
    torch.cuda.set_device(0)
    m = make(n, double_q, L=L, B=B, H=hidden, E=embed, HE=hyper_embed, A=actions)
    batches = [qo.synth_batch(10 * s + n, B, L, n, actions, OBS, SD, max_ep_t=(L + 1 if full else min(L, 3 + s)))
               for s in range(steps)]
    check_train(m, batches, double_q)


@pytest.mark.parametrize("full", [True, False], ids=["full", "short"])
def test_qmix_yaml_shape_matches_oracle(tc_mode, full):
    """qmix.yaml's widths (batch 32, hidden 64, mixing embed 32, hypernet embed 64) at the 2s_vs_1sc sizes that
    scripts/qmix_step.py times (2 agents, 7 actions, obs 26, state 27, episode limit 300): 301-step recurrences, a full
    first embed slot, and both second hypernetwork layers on the tensor cores in mode 1.

    On the tensor cores the magnitude floor is 1e-4 instead of 1e-5.  The weight gradients of those two layers reduce
    over B L = 9600 rows with each fp32 operand carried as two bf16 planes: on an H100 80GB HBM3 (700 W power limit)
    their first-step gradients were
    2.2e-5 (hyper_w1) and 1.6e-5 (hyper_w_final) of the largest gradient from float64, against 3e-7 on the fp32 path
    and 1.4e-7 for the fp32 restatement, while every other gradient (the GRU's included) stayed within 3.7e-6 on both
    paths.  Through the second RMSProp step this left up to 4.3e-5 of the magnitude beyond 8x the fp32 distance
    (hyper_w1/dense_1's slots); the fp32 path stayed within 1.2e-6."""
    torch.cuda.set_device(0)
    n, B, L, nA, obs, sd = 2, 32, 300, 7, 26, 27
    m = make(n, True, L=L, B=B, H=64, E=32, HE=64, A=nA, obs=obs, sd=sd)
    names = [layer[0] for layer in m.hyper.arch["layers"]]
    for name in ("hyper_w1/dense_1", "hyper_w_final/dense_1"):
        assert m.hyper.layer_plan(names.index(name))["tc"], name
    batches = [qo.synth_batch(s, B, L, n, nA, obs, sd, max_ep_t=(L + 1 if full else 60)) for s in range(2)]
    check_train(m, batches, True, floor=1e-4 if tc_mode else 1e-5)


def test_per_sequence_lengths_match_oracle_replayed_and_eager():
    """Every sequence of a batch gets its own length in [0, L + 1], with 0 and L + 1 in the first GRU CTA and the last
    CTA holding one sequence (135 sequences, two per CTA).  The captured graph is replayed with a second set of lengths:
    the kernels read them on the device."""
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    n, B, L = 5, 27, 8
    assert gru_groups(B, n) == 2
    rng = np.random.default_rng(11)

    def batch(seed):
        lens = rng.integers(0, L + 2, size=B * n).astype(np.int32)
        lens[:2] = (0, L + 1)
        lens[-1] = 1 + seed % L
        return dict(qo.synth_batch(seed, B, L, n, A, OBS, SD, max_ep_t=L + 1), seq_len=lens)

    b1, b2, b3 = batch(1), batch(2), batch(3)
    assert not np.array_equal(b2["seq_len"], b3["seq_len"])
    g, e = make(n, L=L, B=B, use_graph=True), make(n, L=L, B=B, use_graph=False)
    replays = capi.lib().xtb_graph_replay_count()
    check_train(e, [b1, b2], True)
    check_train(g, [b1, b2, b3], True)
    assert capi.lib().xtb_graph_replay_count() - replays == 3


TIED = (3, 35, 36)   # lane 3 twice (first and second stride) and lane 4


@pytest.mark.parametrize("double_q,tied", [(True, "eval"), (True, "both"), (False, "target"), (False, "both")])
def test_argmax_ties_under_a_live_mask(double_q, tied):
    """Actions 3, 35 and 36 get a zero dense_1 kernel column and the same bias, above every other action's Q, in the
    eval set, the target set or both: their Q values tie exactly on every row.  Action 3 is unavailable on every other
    step, so the tie is then between lanes 3 and 4, else also within lane 3.  With double Q and the tie in the eval set
    only, the target Q differs between the tied actions, so the tie rule (lowest index, as tf.argmax) decides the loss."""
    torch.cuda.set_device(0)
    n, B, L, nA = 3, 4, 8, 40
    m = make(n, double_q, L=L, B=B, A=nA)
    (ko, ks), (bo, _) = m.agent_vars["dense_1/kernel"], m.agent_vars["dense_1/bias"]
    for flat in {"eval": [m.params], "target": [m.target], "both": [m.params, m.target]}[tied]:
        flat[ko:ko + ks[0] * ks[1]].view(ks)[:, list(TIED)] = 0.0
        flat[bo:bo + nA][list(TIED)] = 20.0
    params_changed(m)
    b = qo.synth_batch(4, B, L, n, nA, OBS, SD, max_ep_t=L + 1)
    av = b["avail"]
    filled = av.sum(-1, keepdims=True) > 0
    av[..., list(TIED)] = np.where(filled, 1.0, 0.0)
    av[:, ::2, :, TIED[0]] = 0.0
    # the restatement's own Q values of the set the target step ranks must tie on enough masked-in rows
    ranked = m.variables(m.params if double_q else m.target, mixer=False)
    with orc.precision("f64"):
        q, _ = qo.agent_forward({k: qo._t(v) for k, v in ranked.items()}, qo._t(b["obs"]), b["seq_len"])
    assert qo.count_ties(q.numpy(), av, b["mask"]) >= 60
    check_train(m, [b], double_q)


def test_zero_hypernetwork_outputs(tc_mode):
    """One output column of hyper_w1 and one of hyper_w_final is exactly 0 on every row (zero kernel column and bias):
    the gradient of |w| there is 0, as TF's Abs gradient and torch's, so those columns must not move."""
    torch.cuda.set_device(0)
    n = 2
    m = make(n)
    cols = (("hyper_w1/dense_1", 5), ("hyper_w_final/dense_1", 3))
    for name, c in cols:
        (ko, ks), (bo, _) = m.mixer_vars[name + "/kernel"], m.mixer_vars[name + "/bias"]
        m.params[ko:ko + ks[0] * ks[1]].view(ks)[:, c] = 0.0
        m.params[bo + c] = 0.0
    params_changed(m)
    w64 = check_train(m, [qo.synth_batch(6, 4, 8, n, A, OBS, SD, max_ep_t=9)], True)
    wd = m.variables(m.params)
    for name, c in cols:
        assert np.all(w64[name + "/kernel"][:, c] == 0) and w64[name + "/bias"][c] == 0
        assert np.all(wd[name + "/kernel"][:, c] == 0) and wd[name + "/bias"][c] == 0, name


def test_models_with_different_gru_widths_train_side_by_side():
    """The GRU kernels' shared-memory opt-in belongs to the kernels, not to a model: creating a model with a narrower
    GRU must not stop one with a wider GRU, created before it, from training."""
    torch.cuda.set_device(0)
    wide, narrow = make(2, H=137), make(2, H=16)
    for s, m in enumerate((wide, narrow)):
        check_train(m, [qo.synth_batch(20 + s, 4, 8, 2, A, OBS, SD, max_ep_t=9)], True)


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


def check_infer(models, w, n, nA, obs, steps=4):
    """infer_actions of every model (all holding the explore weights w) over two episodes against the restatement with
    the hidden state carried; the models must agree bit for bit."""
    rng = np.random.default_rng(5)
    for episode in range(2):
        for m in models:
            m.reset_hidden_state()
        h64 = h32 = None
        for step in range(steps):
            x = rng.normal(size=(1, 1, n, obs)).astype(np.float32)
            qs = [m.infer_actions(x) for m in models]
            assert qs[0].shape == (1, n, nA)
            ref = {}
            for prec in ("f64", "f32"):
                with orc.precision(prec):
                    wt = {k: qo._t(v) for k, v in w.items()}
                    h0 = h64 if prec == "f64" else h32
                    qr, hT = qo.agent_forward(wt, qo._t(x), [1] * n, h0)
                    ref[prec] = qr.numpy().reshape(1, n, nA)
                    if prec == "f64":
                        h64 = hT
                    else:
                        h32 = hT
            close(qs[0], ref["f64"], ref["f32"], "q episode %d step %d" % (episode, step))
            assert all(np.array_equal(q, qs[0]) for q in qs[1:]), (episode, step)


def test_infer_actions_carries_the_hidden_state():
    torch.cuda.set_device(0)
    n = 3
    assert gru_groups(4, n) == 1
    m = make(n)
    b = qo.synth_batch(1, 4, 8, n, A, OBS, SD, max_ep_t=9)
    m.train(*qo.model_args(b))
    m.assign_explore_agent()
    check_infer([m], m.variables(m.explore, mixer=False), n, A, OBS)


# (n_agents, batch): the inference runs with the training shape's sequences per GRU CTA, G = 2 and 8 (32 agents over
# four CTAs), so one CTA carries the hidden states of several agents
@pytest.mark.parametrize("n,B", [(5, 27), (32, 32)])
def test_infer_actions_with_several_sequences_per_gru_cta(n, B):
    torch.cuda.set_device(0)
    assert gru_groups(B, n) == {27: 2, 32: 8}[B]
    m = make(n, L=4, B=B)
    b = qo.synth_batch(1, B, 4, n, A, OBS, SD, max_ep_t=5)
    m.train(*qo.model_args(b))
    m.assign_explore_agent()
    check_infer([m], m.variables(m.explore, mixer=False), n, A, OBS)


def test_explore_scene_matches_train_scene_and_oracle():
    """QMixAlg's explorers build the explore scene (batch 1, episode limit 1): at qmix.yaml's widths, loaded with a
    trained model's explore weights, it must act as the train scene does and as the restatement does."""
    from xingtian_b200.model.qmix import QMixModel
    torch.cuda.set_device(0)
    n, nA, obs, sd = 2, 7, 26, 27
    m = make(n, L=8, B=4, H=64, E=32, HE=64, A=nA, obs=obs, sd=sd)
    m.train(*qo.model_args(qo.synth_batch(3, 4, 8, n, nA, obs, sd, max_ep_t=9)))
    m.assign_explore_agent()
    x = QMixModel(dict(model_config=dict(m.model_config, init_seed=7), scene="explore"))
    assert x.opt is None
    w = m.get_weights()
    x.set_weights(w)
    assert all(np.array_equal(x.get_weights()[k], v) for k, v in w.items())
    check_infer([x, m], x.variables(x.explore, mixer=False), n, nA, obs, steps=6)


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
    for over in (dict(n_actions=256), dict(rnn_hidden_dim=160), dict(rnn_hidden_dim=138), dict(n_agents=33),
                 dict(mixing_embed_dim=129)):
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
