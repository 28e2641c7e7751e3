"""GPU tier: SCCModel's device training step, critic and one-step inference against the float64 restatement
(tests/scc_oracle.py), under test_gpu_qmix.py's bound: 8x the fp32 restatement's distance from float64 plus 1e-5 of the
quantity's magnitude."""
import random

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
import scc_oracle as so
from test_gpu_qmix import close

pytestmark = pytest.mark.gpu

H, A, U = 16, 5, 32


def make(n, groups_map="none", merge="concat", multi=True, L=6, B=3, seed=0, use_graph=True, U=U, mc=2, o=4, actor_clip=5, **over):
    from xingtian_b200.model.scc import SCCModel
    mc_ = dict(gamma=0.99, mixer_grad_norm_clip=5, actor_grad_norm_clip=actor_clip, a_lr=0.0005, c_lr=0.0005, rnn_hidden_dim=H,
               batch_size=B, use_double_q=True, dense_unit_number=U, enable_critic_multi_channel=multi, channel_merge=merge,
               mc_sample_times=mc, map_name=groups_map, n_agents=n, n_actions=A, episode_limit=L,
               state_shape=[5], init_seed=seed, use_cuda_graph=use_graph)
    mc_.update(over)
    mc_.setdefault("obs_shape", o + mc_["n_actions"] + n)
    return SCCModel(dict(model_config=mc_, scene="train"))


def cfg_of(m):
    return dict(n_agents=m.n_agents, n_actions=m.n_actions, multi=m.multi_channel, groups=m.agent_group, merge=m.channel_merge,
                gamma=m.gamma, c_lr=m.c_lr, a_lr=m.a_lr, mixer_clip=m.mixer_grad_norm_clip, actor_clip=m.actor_grad_norm_clip)


def split(m, flat):
    w = m.variables(flat)
    return (OrderedDictSlice(w, m.agent_vars), OrderedDictSlice(w, m.mixer_vars))


def OrderedDictSlice(w, table):
    return {k: w[k] for k in table}


def oracle_run(m, wa, wc, wt, batches, subsets, prec):
    with orc.precision(prec):
        lrn = so.SccLearner(wa, wc, wt, cfg_of(m))
        losses = [lrn.step(b, s) for b, s in zip(batches, subsets)]
        return np.array(losses), lrn.weights(), lrn.slots()


def check_train(m, batches, floor=1e-5):
    wa, wc = split(m, m.params)
    _, wt = split(m, m.target)
    state = random.getstate()
    dev = []
    for b in batches:
        dev.append((np.float32(m.train(*so.model_args(b))), m.mixer_loss, m.actor_loss))
    # the subsets the model drew, replayed from the same `random` state
    random.setstate(state)
    subsets = [m.draw_subsets() if m.n_agents > 2 else None for _ in batches]
    l64, w64, s64 = oracle_run(m, wa, wc, wt, batches, subsets, "f64")
    l32, w32, s32 = oracle_run(m, wa, wc, wt, batches, subsets, "f32")
    close([d[1] for d in dev], l64[:, 0], l32[:, 0], "mixer loss", floor)
    close([d[2] for d in dev], l64[:, 1], l32[:, 1], "actor loss", floor)
    assert all(d[0] == np.float32(d[2]) + np.float32(d[1]) for d in dev)
    wd = m.variables(m.params)
    ms = m.variables(torch.cat([m.opt.m, torch.zeros(m.n_params - m.agent_size, device=m.device)]), mixer=False)
    cm = torch.zeros(m.n_params, device=m.device)
    cv = torch.zeros(m.n_params, device=m.device)
    cm[m.o_mix:], cv[m.o_mix:] = m.critic_opt.m, m.critic_opt.v
    am, av = m.variables(cm), m.variables(cv)
    for k in w64:
        close(wd[k], w64[k], w32[k], k, floor)
        if k in m.agent_vars:
            close(ms[k], s64[k], s32[k], k + " ms", floor)
        else:
            close(am[k], s64[k][0], s32[k][0], k + " adam m", floor)
            close(av[k], s64[k][1], s32[k][1], k + " adam v", floor)
    return w64


@pytest.fixture(params=[1, 0], ids=["tc", "fp32"])
def tc_mode(request):
    from xingtian_b200 import capi
    lib = capi.lib()
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(request.param)
    yield request.param
    lib.xtb_set_tc_mode(old)


# (n_agents, map (grouping), multi-channel, merge, mc, full length, actor clip)
CASES = [(1, "x", True, "concat", 1, True, 5), (2, "x", True, "concat", 1, False, 5), (2, "x", True, "add", 1, True, 5),
         (2, "x", False, None, 1, False, 5), (3, "x", True, "concat", 1, True, 5), (3, "x", True, "add", 3, False, 5),
         (3, "x", False, None, 1, True, 5), (3, "x", False, None, 3, False, 5), (5, "2s3z", True, "concat", 3, True, 5),
         (5, "2s3z", True, "add", 1, False, 5), (5, "2s3z", False, None, 3, True, 5), (9, "1c3s5z", True, "concat", 3, False, 5),
         (10, "MMM2", True, "add", 3, True, 5), (10, "MMM2", True, "concat", 1, False, 5), (2, "x", True, "concat", 1, True, 0),
         (5, "2s3z", False, None, 1, False, -1)]


@pytest.mark.parametrize("n,gmap,multi,merge,mc,full,clip", CASES, ids=["-".join(str(x) for x in c) for c in CASES])
@pytest.mark.parametrize("steps", [1, 3])
def test_train_matches_oracle(n, gmap, multi, merge, mc, full, clip, steps):
    torch.cuda.set_device(0)
    random.seed(100 + n)
    L, B = 6, 3
    m = make(n, gmap, merge or "concat", multi, L=L, B=B, mc=mc, actor_clip=clip)
    batches = [so.synth_batch(10 * s + n, B, L, n, A, 4, max_ep_t=(L + 1 if full else min(L, 3 + s))) for s in range(steps)]
    check_train(m, batches)


def test_widest_critic(tc_mode):
    """U = 512, the widest critic create accepts."""
    torch.cuda.set_device(0)
    random.seed(3)
    m = make(3, "x", "concat", True, U=512)
    check_train(m, [so.synth_batch(1, 3, 6, 3, A, 4, max_ep_t=7)], floor=1e-4 if tc_mode else 1e-5)


@pytest.mark.parametrize("multi", [True, False], ids=["multi", "single"])
def test_scc_yaml_shape_matches_oracle(tc_mode, multi):
    """scc.yaml's widths (batch 32, hidden 64, U 128, mc 3) at the 2s_vs_1sc sizes (2 agents, 7 actions, 26 augmented
    obs, episode limit 300; unverified, SMAC is not in this tree), max_ep_t 60."""
    torch.cuda.set_device(0)
    n, nA, L, B = 2, 7, 300, 32
    m = make(n, "2s_vs_1sc", "concat", multi, L=L, B=B, U=128, mc=3, o=26 - nA - n, A=nA, n_actions=nA, rnn_hidden_dim=64,
             obs_shape=26)
    batches = [so.synth_batch(s, B, L, n, nA, 26 - nA - n, max_ep_t=60) for s in range(2)]
    check_train(m, batches, floor=1e-4 if tc_mode else 1e-5)


def test_credit_methods_and_mixer_output_match_oracle():
    torch.cuda.set_device(0)
    for n, multi, merge in ((2, True, "concat"), (3, True, "add"), (3, False, None), (2, False, None)):
        m = make(n, "x", merge or "concat", multi)
        b = so.synth_batch(2, 3, 6, n, A, 4, max_ep_t=7)
        s = so.critic_states(b["raw_obs"], b["actions"], A)
        _, wc = split(m, m.params)
        ref = {}
        for prec in ("f64", "f32"):
            with orc.precision(prec):
                ref[prec] = so.critic({k: so._t(v) for k, v in wc.items()}, s, cfg_of(m)).numpy()
        close(m.get_mixer_output(s), ref["f64"], ref["f32"], "V")
        D = 4 + A
        random.seed(5)
        dev = (m.get_ex_according_to_mcshap_mask if n > 2 else m.get_ex_according_to_mask)(s, n, 4, A)
        random.seed(5)
        subsets = m.draw_subsets() if n > 2 else None
        for prec in ("f64", "f32"):
            with orc.precision(prec):
                ref[prec] = so.credits({k: so._t(v) for k, v in wc.items()}, s, cfg_of(m), subsets).numpy()
        close(dev.reshape(ref["f64"].shape), ref["f64"], ref["f32"], "credits")
        assert D * n == s.shape[-1]


def test_assign_targets_copies_the_critic_only():
    torch.cuda.set_device(0)
    m = make(3, "x")
    m.train(*so.model_args(so.synth_batch(1, 3, 6, 3, A, 4, max_ep_t=7)))
    agent_t = m.target[:m.agent_size].clone()
    m.assign_targets()
    assert torch.equal(m.target[m.o_mix:], m.params[m.o_mix:])
    assert torch.equal(m.target[:m.agent_size], agent_t) and not torch.equal(agent_t, m.params[:m.agent_size])


def test_graph_replay_matches_eager_with_new_lengths():
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    g, e = make(5, "2s3z", use_graph=True), make(5, "2s3z", use_graph=False)
    replays = capi.lib().xtb_graph_replay_count()
    for s, t in enumerate((3, 7, 5)):
        b = so.synth_batch(s, 3, 6, 5, A, 4, max_ep_t=t)
        random.seed(s)
        lg = g.train(*so.model_args(b))
        random.seed(s)
        le = e.train(*so.model_args(b))
        assert abs(lg - le) <= 1e-5 * max(1.0, abs(le)), (s, lg, le)
    assert capi.lib().xtb_graph_replay_count() - replays == 3
    torch.testing.assert_close(g.params, e.params, rtol=1e-5, atol=1e-7)


def test_infer_actions_and_weights_round_trip_and_explore_scene():
    from xingtian_b200.model.scc import SCCModel
    import qmix_oracle as qo
    torch.cuda.set_device(0)
    n = 3
    m = make(n, "x")
    m.train(*so.model_args(so.synth_batch(1, 3, 6, n, A, 4, max_ep_t=7)))
    m.assign_explore_agent()
    x = SCCModel(dict(model_config=dict(m.model_config, init_seed=7), scene="explore"))
    assert x.opt is None
    w = m.get_weights()
    assert list(w) == ["explore_agent/" + k for k in m.agent_vars]
    x.set_weights(w)
    assert all(np.array_equal(x.get_weights()[k], v) for k, v in w.items())
    rng = np.random.default_rng(5)
    wt = m.variables(m.explore, mixer=False)
    for mm in (m, x):
        mm.reset_hidden_state()
    h64 = h32 = None
    for step in range(4):
        inp = rng.normal(size=(1, 1, n, m.obs_shape)).astype(np.float32)
        qs = [mm.infer_actions(inp) for mm in (m, x)]
        ref = {}
        for prec in ("f64", "f32"):
            with orc.precision(prec):
                qr, hT = qo.agent_forward({k: qo._t(v) for k, v in wt.items()}, qo._t(inp), [1] * n, h64 if prec == "f64" else h32)
                ref[prec] = qr.numpy().reshape(1, n, A)
                if prec == "f64":
                    h64 = hT
                else:
                    h32 = hT
        close(qs[0], ref["f64"], ref["f32"], "q step %d" % step)
        assert np.array_equal(qs[0], qs[1])


def test_rejected_configurations_launch_nothing():
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    lib = capi.lib()
    for over in (dict(n_actions=256), dict(rnn_hidden_dim=138), dict(dense_unit_number=513)):
        with pytest.raises(RuntimeError):
            make(2, "x", **over)
    with pytest.raises(RuntimeError):
        make(33, "x")
    before = lib.xtb_launch_count()
    with pytest.raises(RuntimeError, match="double q"):
        make(2, "x", use_double_q=False)
    with pytest.raises(RuntimeError, match="Channel merge"):
        make(2, "x", merge="max")
    assert lib.xtb_launch_count() == before
    m = make(5, "2s3z")
    before = lib.xtb_launch_count()
    import ctypes as C
    desc = capi.SccDesc()
    desc.batch, desc.episode_limit, desc.n_agents, desc.n_groups, desc.gru_off, desc.head_off = 3, 6, 5, 2, m.gru_off, m.head_off
    desc.group[0], desc.group[1], desc.mc_sample_times = 2, 2, 1       # 4 agents in the groups, not 5
    nets = (C.c_void_p * 2)(*[c.handle.value for c in m.critics])
    h = C.c_void_p()
    assert lib.xtb_scc_create(m.fc1.handle, m.fc2.handle, nets, C.byref(desc), C.byref(h)) == -1
    b = so.synth_batch(0, 3, 6, 5, A, 4, max_ep_t=7)
    with pytest.raises(ValueError):
        m.train(*so.model_args(dict(b, raw_obs=b["raw_obs"][..., :3])))
    assert lib.xtb_launch_count() == before


def test_clip_off_turns_both_clips_off():
    """actor_grad_norm_clip <= 0 turns off the critic's clip too (scc_tf.py:421, 440-448): with a critic clip far below
    every gradient norm, a clipped critic step would leave the restatement's unclipped one behind."""
    torch.cuda.set_device(0)
    random.seed(8)
    for clip in (0, -1):
        m = make(5, "2s3z", actor_clip=clip, mixer_grad_norm_clip=1e-4)
        check_train(m, [so.synth_batch(4, 3, 6, 5, A, 4, max_ep_t=7)])
