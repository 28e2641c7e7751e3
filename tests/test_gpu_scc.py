"""GPU tier: SCCModel's device training step, critic and one-step inference against the float64 restatement
(tests/scc_oracle.py), under test_gpu_qmix.py's bound: 8x the fp32 restatement's distance from float64 plus 1e-5 of the
quantity's magnitude, or 1e-4 where the critic's layers run on the tensor cores at the widths and row counts that need
it (each such test says so)."""
import random

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
import scc_oracle as so
from test_gpu_qmix import check_infer, close, gru_groups

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


def check_train(m, batches, floor=1e-5, slot_floor=None, near_zero=None):
    """Train m on the batches and compare both losses, every variable and the optimisers' slots with the restatement
    (close() with the magnitude floor `floor`, `slot_floor` for the slots if given).

    near_zero (one batch only): TF's first Adam step moves a critic weight by c_lr g / (|g| + 3.2e-7), about c_lr times
    the sign of its gradient g.  Where float64's gradient lies within twice the device's rounding of zero (the device's
    Adam m, itself held to the slot bound, is at least half of float64's m away from it, which covers every sign flip),
    the weight may land up to 2 c_lr from float64.  Those elements, at most the share near_zero of each variable, are
    held to 2 c_lr; the rest to close(): a gradient within half of float64's moves the step by at most 0.17 c_lr."""
    assert near_zero is None or len(batches) == 1
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
    sfloor = floor if slot_floor is None else slot_floor
    for k in w64:
        if k in m.agent_vars:
            close(wd[k], w64[k], w32[k], k, floor)
            close(ms[k], s64[k], s32[k], k + " ms", sfloor)
            continue
        close(am[k], s64[k][0], s32[k][0], k + " adam m", sfloor)
        close(av[k], s64[k][1], s32[k][1], k + " adam v", sfloor)
        m64 = s64[k][0]
        zero = np.zeros(m64.shape, bool) if near_zero is None else (np.abs(am[k] - m64) >= np.abs(m64) / 2) & (am[k] != m64)
        assert zero.mean() <= (near_zero or 0), (k, int(zero.sum()), zero.size)
        close(wd[k][~zero], w64[k][~zero], w32[k][~zero], k, floor)
        assert np.all(np.abs(wd[k][zero] - w64[k][zero]) <= 2 * m.c_lr * (1 + 1e-3)), k
    return w64


@pytest.fixture(params=[1, 0], ids=["tc", "fp32"])
def tc_mode(request):
    from xingtian_b200 import capi
    lib = capi.lib()
    old = lib.xtb_get_tc_mode()
    lib.xtb_set_tc_mode(request.param)
    yield request.param
    lib.xtb_set_tc_mode(old)


def reached(m, batches, subsets):
    """What one train call of m on the batches exercises, for the cases to assert the regime they are named for: the
    head width K (scc_head_grad_kernel's grid covers K + 1 elements, scc_reduce_kernel's K + 2 threads), the
    single-channel credit variants V, the GRU sequences per CTA G, agent bits drawn into the Monte-Carlo subsets and the
    largest action taken."""
    B, L, n = m._B, m._L, m.n_agents
    K = m.mixer_vars["v/kernel"][1][0]
    drawn = [s for s in subsets if s is not None]
    bits = int(np.bitwise_or.reduce(np.concatenate([s.reshape(-1) for s in drawn]))) if drawn else 0
    return dict(K=K, V=m.n_variants, G=gru_groups(B, n), sequences=B * n, BL=B * L, L=L, B=B, o=m.o_shape,
                H=m.rnn_hidden_dim, units=m.dense_unit_number, groups=len(m.agent_group) if m.multi_channel else 0,
                bits_from_16=bits >> 16 != 0, action_from_128=max((int(b["actions"].max()) for b in batches), default=0) >= 128,
                dot_tail=m.dense_unit_number % 32 != 0, loss_in_reduce_block_1=(K + 1) % 128 == 0,
                bias_in_head_grid_y_1=K % 128 == 0 and K > 0, partial_last_chunk=B * L > 64 and B * L % 64 != 0,
                partial_last_step_block=B * L % (256 // 32) != 0,
                tc=any(net.layer_plan(i)["tc"] for net in m.critics for i in range(2)))


# (n_agents, map (grouping), multi-channel, merge, mc, full length, actor clip, then hidden, actions, critic units,
# batch, episode limit, raw obs width and what the case must reach (reached())).  A case's id leaves out the second
# part when it is DEF, the test's defaults.
DEF = (H, A, U, 3, 6, 4)
CASES = [c + DEF + ({},) for c in [
    (1, "x", True, "concat", 1, True, 5), (2, "x", True, "concat", 1, False, 5), (2, "x", True, "add", 1, True, 5),
    (2, "x", False, None, 1, False, 5), (3, "x", True, "concat", 1, True, 5), (3, "x", True, "add", 3, False, 5),
    (3, "x", False, None, 1, True, 5), (3, "x", False, None, 3, False, 5), (5, "2s3z", True, "concat", 3, True, 5),
    (5, "2s3z", True, "add", 1, False, 5), (5, "2s3z", False, None, 3, True, 5), (9, "1c3s5z", True, "concat", 3, False, 5),
    (10, "MMM2", True, "add", 3, True, 5), (10, "MMM2", True, "concat", 1, False, 5), (2, "x", True, "concat", 1, True, 0),
    (5, "2s3z", False, None, 1, False, -1)]]
# - 32 agents, the most create accepts: one 32-channel group (every lane of the step kernel's channel and credit loops
#   busy, K = 1024; test_widest_critic takes it to U = 512); single-channel with 2 n mc = 192 and 68 credit variants,
#   whose subset draws set agent bits 16-31.
# - 255 actions (the most): one-hots wider than 128 columns, actions >= 128 taken.
# - Critic widths off the warp: U = 1, 33 and 100 end scc_dot inside a warp stride; U = 127 (add, single) puts the
#   loss thread K + 1 = 128 in the reduce kernel's second block; concat over 4 x 32 units puts the bias (element K =
#   128) in the head-gradient grid's second y block.
# - GRU widths 1, 17 and 137 (the widest whose weights fit in shared memory at one sequence per CTA).
# - B L = 65, 127 and 129 rows: a partial last 64-row head-gradient chunk and a partial last 8-row step block.
# - 27 x 5 = 135 sequences: two per GRU CTA, one in the last; 32 x 32 = 1024: eight per CTA, the most.
# - Episode limit 1 (the state shift min(t + 1, L - 1) stays on row 0), batch 1, and no raw observation columns.
CASES += [
    (32, "x", True, "concat", 2, True, 5, H, A, U, 3, 6, 4, dict(K=1024)),
    (32, "x", False, None, 3, True, 5, H, A, U, 2, 4, 4, dict(V=192, bits_from_16=True)),
    (17, "x", False, None, 2, False, 5, H, A, U, 3, 6, 4, dict(V=68, bits_from_16=True)),
    (3, "x", True, "add", 1, True, 5, H, 255, U, 3, 6, 4, dict(action_from_128=True)),
    (5, "2s3z", False, None, 3, False, 5, H, 255, U, 3, 6, 4, dict(action_from_128=True, V=30)),
    (3, "x", True, "concat", 3, True, 5, H, A, 1, 3, 6, 4, dict(K=3, dot_tail=True)),
    (5, "2s3z", True, "add", 1, False, 5, H, A, 33, 3, 6, 4, dict(dot_tail=True, groups=2)),
    (3, "x", False, None, 3, True, 5, H, A, 100, 3, 6, 4, dict(dot_tail=True, V=18)),
    (5, "2s3z", True, "add", 2, True, 5, H, A, 127, 3, 6, 4, dict(K=127, loss_in_reduce_block_1=True)),
    (3, "x", False, None, 2, False, 5, H, A, 127, 3, 6, 4, dict(K=127, loss_in_reduce_block_1=True)),
    (4, "x", True, "concat", 1, True, 5, H, A, 32, 3, 6, 4, dict(K=128, bias_in_head_grid_y_1=True)),
    (2, "x", True, "concat", 1, True, 5, 1, A, U, 3, 6, 4, dict(H=1)),
    (3, "x", False, None, 3, False, 5, 17, A, U, 3, 6, 4, dict(H=17)),
    (5, "2s3z", True, "add", 1, True, 5, 137, A, U, 3, 6, 4, dict(H=137, G=1)),
    (5, "2s3z", True, "concat", 1, False, 5, H, A, U, 5, 13, 4, dict(BL=65, partial_last_chunk=True, partial_last_step_block=True)),
    (3, "x", True, "add", 2, True, 5, H, A, U, 1, 127, 4, dict(BL=127, partial_last_chunk=True, partial_last_step_block=True)),
    (3, "x", False, None, 2, False, 5, H, A, U, 3, 43, 4, dict(BL=129, partial_last_chunk=True, partial_last_step_block=True)),
    (5, "2s3z", True, "concat", 1, True, 5, H, A, U, 27, 4, 4, dict(G=2, sequences=135)),
    (32, "x", True, "add", 1, False, 5, H, A, U, 32, 2, 4, dict(G=8, sequences=1024)),
    (3, "x", True, "concat", 2, True, 5, H, A, U, 3, 1, 4, dict(L=1)),
    (2, "x", False, None, 1, True, 5, H, A, U, 1, 6, 4, dict(B=1)),
    (5, "2s3z", True, "concat", 1, True, 5, H, A, U, 3, 6, 0, dict(o=0)),
    (3, "x", False, None, 2, False, 5, H, A, U, 3, 6, 0, dict(o=0, V=12)),
]


def _case_id(c):
    return "-".join(str(x) for x in (c[:7] if c[7:13] == DEF else c[:13]))


@pytest.mark.parametrize("n,gmap,multi,merge,mc,full,clip,hidden,actions,units,B,L,o,want", CASES, ids=[_case_id(c) for c in CASES])
@pytest.mark.parametrize("steps", [1, 3])
def test_train_matches_oracle(n, gmap, multi, merge, mc, full, clip, hidden, actions, units, B, L, o, want, steps):
    torch.cuda.set_device(0)
    random.seed(100 + n)
    m = make(n, gmap, merge or "concat", multi, L=L, B=B, U=units, mc=mc, o=o, actor_clip=clip, rnn_hidden_dim=hidden,
             n_actions=actions)
    batches = [so.synth_batch(10 * s + n, B, L, n, actions, o, max_ep_t=(L + 1 if full else min(L, 3 + s)))
               for s in range(steps)]
    state = random.getstate()
    subsets = [m.draw_subsets() if n > 2 else None for _ in batches]
    random.setstate(state)
    got = reached(m, batches, subsets)
    assert all(got[k] == v for k, v in want.items()), (want, got)
    # the cases above keep the 1e-5 floor; a new case whose critic layers run on the tensor cores (the default mode) is
    # held to their 1e-4 floor, as test_widest_critic is
    check_train(m, batches, floor=1e-4 if want and got["tc"] else 1e-5)


# Agent groupings beyond the built-in maps (at most 3 groups there): the most groups create takes, each of one agent;
# the most groups with uneven sizes over the most agents; one agent beside 31, either way round.
GROUPINGS = {"8x1": [1] * 8, "8-uneven": [5, 1, 7, 2, 6, 3, 4, 4], "1-31": [1, 31], "31-1": [31, 1]}


@pytest.mark.parametrize("merge", ["concat", "add"])
@pytest.mark.parametrize("groups", list(GROUPINGS.values()), ids=list(GROUPINGS))
def test_custom_groupings_match_oracle(monkeypatch, groups, merge):
    from xingtian_b200.model import scc
    torch.cuda.set_device(0)
    monkeypatch.setitem(scc.AGENT_GROUPS, "custom", groups)
    n = sum(groups)
    random.seed(40 + n)
    m = make(n, "custom", merge)
    assert m.agent_group == groups and len(m.critics) == len(groups)
    batches = [so.synth_batch(50 + s, 3, 6, n, A, 4, max_ep_t=7 - s) for s in range(2)]
    floor = 1e-4 if reached(m, batches, [None])["tc"] else 1e-5
    # the critic alone: scc_split_kernel lays the caller's states out group by group
    s = so.critic_states(batches[0]["raw_obs"], batches[0]["actions"], A)
    _, wc = split(m, m.params)
    ref = {}
    for prec in ("f64", "f32"):
        with orc.precision(prec):
            ref[prec] = so.critic({k: so._t(v) for k, v in wc.items()}, s, cfg_of(m)).numpy()
    close(m.get_mixer_output(s), ref["f64"], ref["f32"], "V", floor)
    check_train(m, batches, floor=floor)


def test_widest_critic(tc_mode):
    """U = 512, the widest critic create accepts, with 3 agents and with 32 in one group (a head of K = 16384 units)."""
    torch.cuda.set_device(0)
    random.seed(3)
    m = make(3, "x", "concat", True, U=512)
    check_train(m, [so.synth_batch(1, 3, 6, 3, A, 4, max_ep_t=7)], floor=1e-4 if tc_mode else 1e-5)
    m = make(32, "x", "concat", True, U=512, L=4, B=2)
    assert reached(m, [], [])["K"] == 16384
    check_train(m, [so.synth_batch(2, 2, 4, 32, A, 4, max_ep_t=4)], floor=1e-4 if tc_mode else 1e-5)


# (map, agents, actions, raw obs width, episode limit, multi-channel, merge, mc, max_ep_t of each batch, what the case
# must reach (reached()), and on the tensor cores the slot floor and the near-zero share (check_train()))
SMAC = [("2s_vs_1sc", 2, 7, 26 - 7 - 2, 300, True, "concat", 3, (60, 60), {}, None, None),
        ("2s_vs_1sc", 2, 7, 26 - 7 - 2, 300, False, "concat", 3, (60, 60), {}, None, None),
        ("2s3z", 5, 11, 80, 120, True, "concat", 3, (121,), dict(groups=2, G=2), 1e-4, 0.01),
        ("2s3z", 5, 11, 80, 120, False, "concat", 3, (121,), dict(V=30, G=2), 1e-4, 0.01),
        ("MMM2", 10, 18, 176, 180, True, "add", 1, (181,), dict(groups=3, G=3), 1e-4, 0.01)]


@pytest.mark.parametrize("case", SMAC, ids=["multi", "single", "2s3z-multi", "2s3z-single", "MMM2-add"])
def test_scc_yaml_shape_matches_oracle(tc_mode, case):
    """scc.yaml's widths (batch 32, hidden 64, U 128) at SMAC map sizes, which are unverified (SMAC is not in this tree):
    2s_vs_1sc (2 agents, 7 actions, 26 augmented obs, episode limit 300) with max_ep_t 60, two steps; 2s3z as
    scripts/scc_step.py times it (5 agents in groups [2, 3], 11 actions, raw obs 80, episode limit 120), one full batch
    with both critics: the Monte-Carlo Shapley credits (mc 3) at a training size and 160 GRU sequences, two per CTA;
    MMM2 (10 agents in groups [1, 2, 7], 18 actions, raw obs 176, episode limit 180) with the add merge and mc 1, one
    full batch, because the restatement's literal credits evaluate every channel of the critic 2 n mc times.

    On the tensor cores the magnitude floor is 1e-4 instead of 1e-5, as for QMIX's full-size case
    (test_gpu_qmix.test_qmix_yaml_shape_matches_oracle): the critic layers' weight gradients reduce over thousands of
    rows with each fp32 operand carried as two bf16 planes.  The 2s3z and MMM2 steps also allow for TF Adam's first step,
    about c_lr times the sign of the gradient (check_train's near_zero): a first-layer critic weight whose float64
    gradient lies within the tensor cores' rounding of zero may land up to 2 c_lr from float64.  On an H100 80GB HBM3
    (700 W power limit) both losses stayed within 0.06 of their 1e-5 bound, no first-layer unit took the other ReLU
    branch than in float64 on the single-channel critic, and the Adam slots stayed within 0.8 of the 1e-4 floor.  The
    first-layer kernels held 18 and 5 such elements (2s3z multi-channel, 3 of each with the other sign), 227 of 58240
    (2s3z single-channel, 64 with the other sign) and 1 and 48 (MMM2, 9 with the other sign), up to 9.96e-4 (2 c_lr = 1e-3)
    from float64; every other weight stayed within 0.19 of its 1e-4 bound.  The share allowed is 1%."""
    torch.cuda.set_device(0)
    gmap, n, nA, o, L, multi, merge, mc, lengths, want, tc_slot_floor, tc_near_zero = case
    B = 32
    random.seed(60 + n)
    m = make(n, gmap, merge, multi, L=L, B=B, U=128, mc=mc, o=o, n_actions=nA, rnn_hidden_dim=64, obs_shape=o + nA + n)
    batches = [so.synth_batch(s, B, L, n, nA, o, max_ep_t=t) for s, t in enumerate(lengths)]
    state = random.getstate()
    subsets = [m.draw_subsets() if n > 2 else None for _ in batches]
    random.setstate(state)
    got = reached(m, batches, subsets)
    assert all(got[k] == v for k, v in want.items()), (want, got)
    if tc_mode:
        check_train(m, batches, floor=1e-4, slot_floor=tc_slot_floor, near_zero=tc_near_zero)
    else:
        check_train(m, batches)


def test_credit_methods_and_mixer_output_match_oracle():
    """Both credit methods and the critic, with 17 agents among the cases: the Monte-Carlo credit method builds its
    masks on the host from `random`'s draws, which then zero agent 16's action part, and evaluates them through
    get_mixer_output."""
    torch.cuda.set_device(0)
    for n, multi, merge in ((2, True, "concat"), (3, True, "add"), (3, False, None), (2, False, None), (17, True, "concat"),
                            (17, False, None)):
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
        assert n < 17 or reached(m, [b], [subsets])["bits_from_16"]
        for prec in ("f64", "f32"):
            with orc.precision(prec):
                ref[prec] = so.credits({k: so._t(v) for k, v in wc.items()}, s, cfg_of(m), subsets).numpy()
        close(dev.reshape(ref["f64"].shape), ref["f64"], ref["f32"], "credits")
        assert D * n == s.shape[-1]


@pytest.mark.parametrize("multi", [True, False], ids=["multi", "single"])
def test_mixer_output_over_more_rows_than_a_batch(multi):
    """get_mixer_output evaluates at most B L rows per device call: 2.5 B L rows under two leading axes take two full
    calls and a half one, each row count with its own captured graph; replayed, and eager, the values must not change."""
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    lib = capi.lib()
    n = 5
    g, e = make(n, "2s3z", "concat", multi, use_graph=True), make(n, "2s3z", "concat", multi, use_graph=False)
    assert torch.equal(g.params, e.params)
    s = np.random.default_rng(4).normal(size=(5, 9, n * (4 + A)))
    assert s.shape[0] * s.shape[1] == 2.5 * g._B * g._L
    _, wc = split(g, g.params)
    ref = {}
    for prec in ("f64", "f32"):
        with orc.precision(prec):
            ref[prec] = so.critic({k: so._t(v) for k, v in wc.items()}, s, cfg_of(g)).numpy()
    replays = [g.get_mixer_output(s)]
    before = lib.xtb_graph_replay_count()
    replays.append(g.get_mixer_output(s))
    assert lib.xtb_graph_replay_count() - before == 3
    before = lib.xtb_graph_replay_count()
    eager = e.get_mixer_output(s)
    assert lib.xtb_graph_replay_count() == before
    assert eager.shape == s.shape[:-1] + (1,)
    close(eager, ref["f64"], ref["f32"], "V")
    assert all(np.array_equal(v, eager) for v in replays)


@pytest.mark.parametrize("multi,merge", [(True, "concat"), (True, "add"), (False, None)], ids=["concat", "add", "single"])
def test_dead_critic_unit_stays_put(multi, merge):
    """Unit k of every second critic layer has a zero kernel column and a zero bias, in the eval and in the target
    critic: its output is exactly 0 on every row, where TF's ReLU gradient is 0.  Its weights, their Adam moments and
    the head rows it feeds (every channel's with concat) must stay exactly as they were."""
    torch.cuda.set_device(0)
    n, k = 5, 7
    random.seed(9)
    m = make(n, "2s3z", merge or "concat", multi)
    dead = [name for name in m.mixer_vars if name.endswith("dense_1/kernel") or name.endswith("dense_1/bias")]
    assert len(dead) == 2 * len(m.critics)
    for flat in (m.params, m.target):
        for name in dead:
            o, shape = m.mixer_vars[name]
            flat[o:o + int(np.prod(shape))].view(shape)[..., k] = 0.0
    for net in m.critics:
        net.params_changed()
    head = m.variables(m.params)["v/kernel"]
    rows = [c * U + k for c in range(n)] if merge == "concat" else [k]
    check_train(m, [so.synth_batch(6, 3, 6, n, A, 4, max_ep_t=7)])
    w = m.variables(m.params)
    cm = torch.zeros(m.n_params, device=m.device)
    cv = torch.zeros(m.n_params, device=m.device)
    cm[m.o_mix:], cv[m.o_mix:] = m.critic_opt.m, m.critic_opt.v
    am, av = m.variables(cm), m.variables(cv)
    for name in dead:
        assert np.all(w[name][..., k] == 0) and np.all(am[name][..., k] == 0) and np.all(av[name][..., k] == 0), name
    assert np.array_equal(w["v/kernel"][rows], head[rows])
    assert np.all(am["v/kernel"][rows] == 0) and np.all(av["v/kernel"][rows] == 0)
    assert not np.array_equal(w["v/kernel"], head)


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


def test_infer_actions_with_eight_sequences_per_gru_cta():
    """The one-step inference runs with the training shape's sequences per GRU CTA: 32 episodes of 32 agents give
    eight, so one CTA carries the hidden states of eight agents from step to step."""
    torch.cuda.set_device(0)
    n, B = 32, 32
    assert gru_groups(B, n) == 8
    m = make(n, "x", L=2, B=B)
    check_infer([m], m.variables(m.explore, mixer=False), n, A, m.obs_shape)


@pytest.mark.parametrize("multi", [True, False], ids=["multi", "single"])
def test_step_is_bitwise_reproducible(multi):
    """Two models from the same seed, trained once on the same batch and `random` state: both losses (the step
    kernel's per-block partials, summed in block order) and the head's weights after the step (its gradient from the
    head-gradient kernel's 64-row chunks, summed in chunk order) repeat bit for bit.  108 rows: 14 step blocks, two
    chunks.  The engine's split-K weight gradients of the critic and agent layers are not part of this."""
    torch.cuda.set_device(0)
    n, B, L = 5, 27, 4
    b = so.synth_batch(7, B, L, n, A, 4, max_ep_t=L + 1)
    out = []
    for _ in range(2):
        m = make(n, "2s3z", "concat", multi, L=L, B=B, seed=3, mc=3)
        random.seed(12)
        m.train(*so.model_args(b))
        w = m.variables(m.params)
        out.append((m.mixer_loss, m.actor_loss, w["v/kernel"], w["v/bias"]))
    assert out[0][:2] == out[1][:2]
    assert np.array_equal(out[0][2], out[1][2]) and np.array_equal(out[0][3], out[1][3])


def test_scc_and_qmix_with_different_gru_widths_train_side_by_side():
    """The GRU kernels' shared-memory opt-in is shared by the SCC and the QMIX objects: creating one with a narrower GRU
    must not stop the other, created before it with a wider GRU, from training."""
    import qmix_oracle as qo
    import test_gpu_qmix as tq
    torch.cuda.set_device(0)
    random.seed(21)
    scc_wide, qmix_narrow = make(3, "x", rnn_hidden_dim=137), tq.make(2, H=16)
    qmix_wide, scc_narrow = tq.make(2, H=137), make(3, "x", rnn_hidden_dim=8)
    for s, m in enumerate((scc_wide, scc_narrow)):
        check_train(m, [so.synth_batch(30 + s, 3, 6, 3, A, 4, max_ep_t=7)])
    for s, m in enumerate((qmix_wide, qmix_narrow)):
        tq.check_train(m, [qo.synth_batch(40 + s, 4, 8, 2, tq.A, tq.OBS, tq.SD, max_ep_t=9)], True)


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
    m, single = make(5, "2s3z"), make(5, "2s3z", multi=False, mc=3)
    before = lib.xtb_launch_count()
    import ctypes as C

    def create(model, batch=3, episode_limit=6, n_groups=None, group=(2, 3), mc_sample_times=1):
        """xtb_scc_create on model's nets with model's descriptor but the given fields -> its error message."""
        desc = capi.SccDesc()
        desc.batch, desc.episode_limit, desc.n_agents, desc.gru_off, desc.head_off = batch, episode_limit, 5, model.gru_off, model.head_off
        desc.n_groups = len(model.critics) if model.multi_channel and n_groups is None else n_groups or 0
        for j, g in enumerate(group):
            desc.group[j] = g
        desc.mc_sample_times = mc_sample_times
        nets = (C.c_void_p * len(model.critics))(*[c.handle.value for c in model.critics])
        h = C.c_void_p()
        assert lib.xtb_scc_create(model.fc1.handle, model.fc2.handle, nets, C.byref(desc), C.byref(h)) == -1
        return lib.xtb_last_error().decode()

    assert "4 agents" in create(m, group=(2, 2))
    assert "n_groups 9" in create(m, n_groups=9)
    assert "group 1 has 0 agents" in create(m, n_groups=3, group=(2, 0, 3))
    assert "mc_sample_times 0" in create(single, mc_sample_times=0)
    # B L n max(D, U) V floats of the single-channel credit rows: 32 x 7000 x 5 x 32 x 30 is just over 2^30, and an
    # episode limit of 6990 is within it (and then too many rows for the nets)
    assert "batch too large" in create(single, batch=32, episode_limit=7000, mc_sample_times=3)
    assert "batch too large" not in create(single, batch=32, episode_limit=6990, mc_sample_times=3)
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
