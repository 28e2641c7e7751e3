"""GPU tier: acting for many environments of one QMIX / SCC agent network in one device call (QMixModel.act,
xtb_qmix_act / xtb_scc_act): each environment's Q against the float64 restatement with its own carried hidden state
(test_gpu_qmix.py's bound), the actions bit for bit against the host selector's rule on the same uniforms (given, or the
documented Philox draws), the independence of the environments, the agreement with the one-environment infer_actions,
and the training step of a model built for many environments."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
import qmix_act_oracle as qa
import qmix_oracle as qo
import scc_oracle as so
import test_gpu_qmix as tq
import test_gpu_scc as ts
from test_gpu_qmix import close, gru_groups

pytestmark = pytest.mark.gpu

O = 6   # raw observation width of the QMIX models


def qmix(n, N, last=True, ident=True, **over):
    over.setdefault("obs", O + (over.get("A", tq.A) if last else 0) + (n if ident else 0))
    return tq.make(n, act_envs=N, obs_last_action=last, obs_agent_id=ident, **over)


def scc(n, N, last=True, ident=True, **over):
    return ts.make(n, "none", act_envs=N, obs_last_action=last, obs_agent_id=ident, **over)


def trained(kind, n, N, last=True, ident=True, **over):
    """A model after one training step, its explore agent synced from the eval set."""
    if kind == "qmix":
        m = qmix(n, N, last, ident, **over)
        m.train(*qo.model_args(qo.synth_batch(1, 4, 8, n, tq.A, m.obs_shape, tq.SD, max_ep_t=9)))
    else:
        m = scc(n, N, last, ident, **over)
        m.train(*so.model_args(so.synth_batch(1, 3, 6, n, ts.A, 4, max_ep_t=7)))
    m.assign_explore_agent()
    return m


def q_of(m, N):
    """The Q values of the last act, read from fc2's output tensor -> [N, n, A]."""
    n, A = m.n_agents, m.n_actions
    return m.fc2.tensor("dense_1").reshape(-1)[:N * n * A].cpu().numpy().reshape(N, n, A)


def philox_uniforms(seed, N, n, k):
    """(u0, u1) of agent row (e, a) at per-slot counter k[e]: words (0, 1) and (2, 3) of Philox4x32-10 on counter
    (a, e, k) with key seed, 53 bits each -> [N, 2, n]."""
    ctr = np.zeros((N, n, 4), np.uint32)
    k = np.asarray(k, np.uint64)
    ctr[..., 0] = np.arange(n, dtype=np.uint32)[None]
    ctr[..., 1] = np.arange(N, dtype=np.uint32)[:, None]
    ctr[..., 2] = (k & np.uint64(0xffffffff)).astype(np.uint32)[:, None]
    ctr[..., 3] = (k >> np.uint64(32)).astype(np.uint32)[:, None]
    w = orc.philox4x32_10(ctr.reshape(-1, 4), np.array([seed & 0xffffffff, seed >> 32], np.uint32)).reshape(N, n, 4)
    u = lambda a, b: ((w[..., a] >> 5).astype(np.float64) * 67108864.0 + (w[..., b] >> 6).astype(np.float64)) / 9007199254740992.0
    return np.stack([u(0, 1), u(2, 3)], axis=1)


def sparse_avail(rng, N, n, A):
    """Random 0/1 masks with about a third of the actions available, one row in five with a single one, and weights up
    to 3 on some rows."""
    av = (rng.random((N, n, A)) < 0.35).astype(np.int32)
    av[np.arange(N)[:, None], np.arange(n)[None], rng.integers(0, A, size=(N, n))] = 1
    one = rng.random((N, n)) < 0.2
    av[one] = 0
    av[one, rng.integers(0, A)] = 1
    heavy = rng.random((N, n)) < 0.1
    av[heavy] *= rng.integers(1, 4, size=(int(heavy.sum()), A)).astype(np.int32)
    av[heavy, 0] = np.maximum(av[heavy, 0], 1)
    return av


def agent_inputs(obs, prev, reset, A, last, ident):
    """build_inputs for one step: obs, the previous action's one-hot (zeros after a reset), the agent's one-hot."""
    N, n, _ = obs.shape
    parts = [obs]
    if last:
        oh = np.zeros((N, n, A), np.float32)
        if prev is not None:
            for e in range(N):
                if not reset[e]:
                    oh[e, np.arange(n), prev[e]] = 1.0
        parts.append(oh)
    if ident:
        parts.append(np.tile(np.eye(n, dtype=np.float32)[None], (N, 1, 1)))
    return np.concatenate(parts, -1)


def drive(m, N, steps, seed, eps=0.3, given=False, check_q=True, obs_fn=None, avail_fn=None):
    """`steps` act calls on environments 0..N-1, every environment reset at step 0 and then every third step, staggered
    by its slot.  Each call's actions must be the NumPy selector's on the downloaded Q and the same uniforms (given ones,
    or Philox's at the slot's counter) and, with check_q, each environment's Q must be within close() of the float64
    restatement with its own carried hidden state.  -> [(actions, q)] per step."""
    rng = np.random.default_rng(seed)
    n, A, H = m.n_agents, m.n_actions, m.rnn_hidden_dim
    w = m.variables(m.explore, mixer=False)
    h = {}
    prev, out = None, []
    k = m.act_counter.cpu().numpy().astype(np.uint64)[:N]
    for step in range(steps):
        reset = np.ones(N, bool) if step == 0 else (np.arange(N) + step) % 3 == 0
        obs = obs_fn(step, N) if obs_fn else rng.normal(size=(N, n, m.act_obs_dim)).astype(np.float32)
        avail = avail_fn(step, N) if avail_fn else sparse_avail(rng, N, n, A)
        u = rng.random((N, 2, n)) if given else None
        acts = m.act(obs, avail, reset, eps, u)
        q = q_of(m, N)
        if not given:
            k = k + np.uint64(1)
            u = philox_uniforms(m._act_seed, N, n, k)
        assert acts.dtype == np.int32 and acts.shape == (N, n)
        assert np.array_equal(acts, qa.select_actions(q, avail, np.broadcast_to(eps, (N,)), u)), step
        if check_q:
            x = agent_inputs(obs, prev, reset, A, m.obs_last_action, m.obs_agent_id)
            ref = {}
            for prec in ("f64", "f32"):
                with orc.precision(prec):
                    h0 = h.get(prec, qo._t(np.zeros((N * n, H))))
                    h0 = torch.where(torch.as_tensor(np.repeat(reset, n))[:, None], torch.zeros_like(h0), h0)
                    qr, h[prec] = qo.agent_forward({kk: qo._t(v) for kk, v in w.items()}, qo._t(x[:, None]), [1] * N * n, h0)
                    ref[prec] = qr.numpy().reshape(N, n, A)
            close(q, ref["f64"], ref["f32"], "q step %d" % step)
        prev = acts
        out.append((acts, q))
    return out


# (environments, agents): N n sequences give 1, 1, 2 and 8 sequences per GRU CTA
SIZES = [(1, 3), (3, 3), (64, 3), (300, 4)]


@pytest.mark.parametrize("switches", [(True, True), (False, False), (True, False)], ids=["last-id", "obs-only", "last"])
@pytest.mark.parametrize("N,n", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("kind", ["qmix", "scc"])
def test_q_and_actions_match_oracle(kind, N, n, switches):
    torch.cuda.set_device(0)
    assert gru_groups(N, n) == {1: 1, 3: 1, 64: 2, 300: 8}[N]
    m = trained(kind, n, N, *switches)
    drive(m, N, 7, seed=N + n)


def test_given_uniforms_forced_ties_and_greedy():
    """A zero fc2 kernel and a bias shared by actions 1, 3 and 4 (above the others) make every row's Q tie exactly; the
    sparse masks decide which of them is the first available.  Given uniforms at epsilon 0.5, then greedy (0)."""
    torch.cuda.set_device(0)
    n, N = 3, 40
    m = trained("qmix", n, N)
    (ko, ks), (bo, _) = m.agent_vars["dense_1/kernel"], m.agent_vars["dense_1/bias"]
    m.explore[ko:ko + ks[0] * ks[1]] = 0.0
    m.explore[bo:bo + tq.A].copy_(torch.tensor([0.0, 2.0, -1.0, 2.0, 2.0]))
    for eps in (0.5, 0.0):
        for acts, q in drive(m, N, 4, seed=3, eps=eps, given=True):
            assert np.all(q[..., 1] == q[..., 3]) and np.all(q[..., 1] == q[..., 4]) and np.all(q[..., 1] > q[..., 0])


def test_philox_draws_do_not_depend_on_n_neighbours_or_graph_replay():
    """Environment e's actions and Q, with Philox draws, are the same whether 64 or 5 environments are stepped, whatever
    its neighbours see, eagerly or graph-replayed; the same seed repeats the draws."""
    torch.cuda.set_device(0)
    n, steps = 3, 6
    base = np.random.default_rng(0)
    obs = base.normal(size=(steps, 64, n, O)).astype(np.float32)
    avail = np.stack([sparse_avail(base, 64, n, tq.A) for _ in range(steps)])
    other = np.random.default_rng(1).normal(size=obs.shape).astype(np.float32)
    other[:, :5] = obs[:, :5]

    def run(N, use_graph=True, o=obs):
        m = qmix(n, 64, seed=4, use_graph=use_graph)
        return drive(m, N, steps, seed=9, eps=0.4, check_q=False, obs_fn=lambda s, N: o[s, :N], avail_fn=lambda s, N: avail[s, :N]), m

    full, m1 = run(64)
    few, _ = run(5)
    eager, _ = run(64, use_graph=False)
    nbrs, _ = run(64, o=other)
    again, m2 = run(64)
    assert m1._act_seed == m2._act_seed
    for s in range(steps):
        assert np.array_equal(full[s][0][:5], few[s][0])
        # a different number of rows may sum the dense layers in another order: within fp32 rounding
        np.testing.assert_allclose(full[s][1][:5], few[s][1], rtol=1e-5, atol=1e-6)
        assert np.array_equal(full[s][0], eager[s][0]) and np.array_equal(full[s][1], eager[s][1])
        assert np.array_equal(full[s][0][:5], nbrs[s][0][:5]) and np.array_equal(full[s][1][:5], nbrs[s][1][:5])
        assert np.array_equal(full[s][0], again[s][0]) and np.array_equal(full[s][1], again[s][1])
    other_seed = qmix(n, 64, seed=5)
    diff = drive(other_seed, 64, 2, seed=9, eps=0.4, check_q=False, obs_fn=lambda s, N: obs[s, :N], avail_fn=lambda s, N: avail[s, :N])
    assert not np.array_equal(diff[1][0], full[1][0])


def test_epsilon_one_is_uniform_and_zero_is_greedy():
    """Epsilon 1 with actions 1, 4 and 6 of 7 available: 20480 Philox draws, chi-square against uniform over the three
    below 20 (2 degrees of freedom; p ~ 5e-5).  Epsilon 0: the masked argmax."""
    torch.cuda.set_device(0)
    n, N, A = 4, 256, 7
    m = qmix(n, N, A=A, obs=O + A + n)
    mask = np.zeros((N, n, A), np.int32)
    mask[..., [1, 4, 6]] = 1
    rng = np.random.default_rng(2)
    counts = np.zeros(A, np.int64)
    for step in range(20):
        acts = m.act(rng.normal(size=(N, n, O)).astype(np.float32), mask, np.full(N, step == 0), 1.0)
        counts += np.bincount(acts.reshape(-1), minlength=A)
    assert counts.sum() == 20 * N * n and counts[[0, 2, 3, 5]].sum() == 0
    expect = counts.sum() / 3.0
    chi2 = float(((counts[[1, 4, 6]] - expect) ** 2 / expect).sum())
    assert chi2 < 20.0, (counts, chi2)
    acts = m.act(rng.normal(size=(N, n, O)).astype(np.float32), mask, np.zeros(N, bool), 0.0)
    q = q_of(m, N)
    assert np.array_equal(acts, np.where(mask > 0, q, -np.inf).argmax(-1))


def test_agrees_with_infer_actions_and_scc_with_qmix():
    """One environment's Q from act equals infer_actions' bit for bit: with one environment both run fc1, the GRU and
    fc2 on the same n rows through the same kernels.  Stepped among 64 environments the dense layers see 64 n rows (the
    GEMM may split its reduction differently), so there it is compared within close().  SCC's act equals QMIX's bit for
    bit with the same agent weights."""
    torch.cuda.set_device(0)
    n = 3
    m = trained("qmix", n, 64, H=ts.H, obs=4 + ts.A + n)
    w = m.variables(m.explore, mixer=False)
    s = trained("scc", n, 64)
    s.set_weights(m.get_weights())
    rng = np.random.default_rng(8)
    m.reset_hidden_state()
    prev, h64, h32 = None, None, None
    for step in range(5):
        obs = rng.normal(size=(64, n, m.act_obs_dim)).astype(np.float32)
        avail = sparse_avail(rng, 64, n, m.n_actions)
        reset = np.full(64, step == 0)
        x = agent_inputs(obs[:1], prev, reset[:1], m.n_actions, True, True)
        q_inf = m.infer_actions(x[None])[0]
        u = rng.random((64, 2, n))
        a64 = m.act(obs, avail, reset, 0.2, u)
        q64 = q_of(m, 64)
        a64s = s.act(obs, avail, reset, 0.2, u)
        assert np.array_equal(a64, a64s) and np.array_equal(q64, q_of(s, 64))
        ref = {}
        for prec in ("f64", "f32"):
            with orc.precision(prec):
                qr, hT = qo.agent_forward({k: qo._t(v) for k, v in w.items()}, qo._t(x[:, None]), [1] * n, h64 if prec == "f64" else h32)
                ref[prec] = qr.numpy().reshape(n, -1)
                if prec == "f64":
                    h64 = hT
                else:
                    h32 = hT
        close(q64[0], ref["f64"], ref["f32"], "act among 64, step %d" % step)
        close(q_inf, ref["f64"], ref["f32"], "infer_actions, step %d" % step)
        prev = a64[:1]
    # one environment: the same rows through the same kernels
    m1 = trained("qmix", n, 1)
    m1.reset_hidden_state()
    prev = None
    for step in range(5):
        obs = rng.normal(size=(1, n, m1.act_obs_dim)).astype(np.float32)
        avail = sparse_avail(rng, 1, n, m1.n_actions)
        x = agent_inputs(obs, prev, [step == 0], m1.n_actions, True, True)
        q_inf = m1.infer_actions(x[None])[0]
        prev = m1.act(obs, avail, [step == 0], 0.2, rng.random((1, 2, n)))
        assert np.array_equal(q_of(m1, 1)[0], q_inf), step


def test_training_is_unchanged_by_act_envs():
    """A model built for 256 acting environments trains bit for bit as the default one: loss, Q gradients and weights."""
    torch.cuda.set_device(0)
    n = 3
    a, b = tq.make(n, seed=2), tq.make(n, seed=2, act_envs=256)
    assert b.fc1.max_batch == 256 * n > a.fc1.max_batch
    for s in range(2):
        batch = qo.synth_batch(30 + s, 4, 8, n, tq.A, tq.OBS, tq.SD, max_ep_t=9)
        la, lb = a.train(*qo.model_args(batch)), b.train(*qo.model_args(batch))
        assert la == lb
        R = 4 * 9 * n * tq.A
        assert torch.equal(a.fc2.tensor_grad("dense_1").reshape(-1)[:R], b.fc2.tensor_grad("dense_1").reshape(-1)[:R])
        assert torch.equal(a.params, b.params) and torch.equal(a.grads, b.grads)


@pytest.mark.parametrize("kind", ["qmix", "scc"])
def test_rejected_arguments_launch_nothing(kind):
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    lib = capi.lib()
    n, N = 2, 4
    m = qmix(n, N) if kind == "qmix" else scc(n, N)
    fn = getattr(lib, m._native + "_act")
    io = m._act_io
    p = lambda t: C.c_void_p(t.data_ptr())
    good = [m.handle, p(m.explore), N, 1, 1, p(io["obs"]), p(io["avail"]), p(io["reset"]), p(io["epsilon"]), C.c_void_p(0), 7,
            p(m.act_counter), p(m.act_hidden), p(m.act_last), p(io["actions"]), 0, None]
    before = lib.xtb_launch_count()
    for i, v in [(2, N + 1), (2, 0), (1, C.c_void_p(0)), (5, C.c_void_p(0)), (6, C.c_void_p(0)), (11, C.c_void_p(0)),
                 (12, C.c_void_p(0)), (14, C.c_void_p(0)), (0, C.c_void_p(0))]:
        args = list(good)
        args[i] = v
        assert fn(*args) == -1, i
        assert lib.xtb_last_error()
    args = list(good)
    args[2] = N + 1
    assert fn(*args) == -1 and b"act_envs" in lib.xtb_last_error()
    assert lib.xtb_launch_count() == before
    dev = dict(device=m.act_hidden.device)
    with pytest.raises(ValueError):
        m.act_device(torch.zeros(N + 1, n, m.act_obs_dim, **dev), torch.ones(N + 1, n, m.n_actions, dtype=torch.int32, **dev),
                     torch.zeros(N + 1, dtype=torch.int32, **dev), torch.zeros(N + 1, dtype=torch.float64, **dev),
                     out=torch.zeros(N + 1, n, dtype=torch.int32, **dev))
    with pytest.raises(ValueError):
        m.act_device(io["obs"], io["avail"].float(), io["reset"], io["epsilon"])
    with pytest.raises(ValueError):
        m.act(np.zeros((N + 1, n, m.act_obs_dim)), np.ones((N + 1, n, m.n_actions), np.int32), np.zeros(N + 1), 0.0)
    assert lib.xtb_launch_count() == before
    # a model too small for its act_envs is refused at create
    desc = capi.QmixDesc()
    if kind == "qmix":
        desc.batch, desc.episode_limit, desc.n_agents, desc.gamma, desc.gru_off, desc.act_envs = 4, 8, n, 0.99, m.gru_off, 10 ** 6
        h = C.c_void_p()
        assert lib.xtb_qmix_create(m.fc1.handle, m.fc2.handle, m.hyper.handle, C.byref(desc), C.byref(h)) == -1
        assert b"act_envs" in lib.xtb_last_error()


def test_predict_with_selector_envs_matches_predict_with_selector():
    """QMixAlg with one environment: predict_with_selector_envs on selector_uniforms draws the host selector's numbers,
    so a seeded session over whole episodes picks the same actions as predict_with_selector; selector.epsilon ends the
    same.  Then N environments with per-environment t_env: the epsilon schedule per environment."""
    from xingtian_b200.algorithm.qmix import EpisodeBatch, QMixAlg
    torch.cuda.set_device(0)
    n, A, obs_dim, limit = 2, 7, 26, 12
    env_attr = dict(n_agents=n, n_actions=A, state_shape=27, obs_shape=obs_dim, episode_limit=limit)
    alg_config = dict(batch_size=4, buffer_size=8, epsilon_anneal_time=40, epsilon_finish=0.05, epsilon_start=1.0, obs_agent_id=True,
                      obs_last_action=True, target_update_interval=3, env_attr=env_attr, instance_num=1, agent_num=1)
    mc = dict(gamma=0.99, lr=0.0005, n_agents=n, rnn_hidden_dim=64, episode_limit=limit, n_actions=A, batch_size=4, state_shape=[27],
              mixing_embed_dim=32, hypernet_embed=64, init_seed=3, act_envs=8)
    alg = QMixAlg({"actor": {"model_name": "QMixModel", "model_config": mc}}, alg_config, scene="explore")
    rng = np.random.default_rng(4)
    episodes = []
    for i in range(4):
        T = int(rng.integers(3, limit + 1))
        episodes.append((rng.normal(size=(T, n, obs_dim)).astype(np.float32), sparse_avail(rng, T, n, A)))

    def host():
        out, t_env = [], 0
        for obs, avail in episodes:
            alg.reset_hidden_state()
            ep = EpisodeBatch(alg.scheme, alg.groups, 1, limit + 1, preprocess=alg.preprocess)
            for t in range(len(obs)):
                ep.update({"obs": obs[t][None], "avail_actions": avail[t][None]}, ts=t)
                a = alg.predict_with_selector(ep, t, t_env, test_mode=t_env > 30)
                ep.update({"actions": a}, ts=t, mark_filled=False)
                out.append(np.asarray(a).reshape(n))
                t_env += 1
        return np.array(out), alg.selector.epsilon

    def device():
        out, t_env = [], 0
        for obs, avail in episodes:
            for t in range(len(obs)):
                a = alg.predict_with_selector_envs(obs[t][None], avail[t][None], [t == 0], t_env, t_env > 30,
                                                   uniforms=alg.selector_uniforms(1, n))
                out.append(a.reshape(n))
                t_env += 1
        return np.array(out), alg.selector.epsilon

    np.random.seed(21)
    want, eps_h = host()
    after = np.random.rand()
    np.random.seed(21)
    got, eps_d = device()
    assert np.random.rand() == after
    assert np.array_equal(got, want) and eps_d == eps_h
    assert len(set(map(tuple, want))) > 3
    # N environments, each with its own t_env: epsilon of its own schedule point (given uniforms decide)
    N = 8
    t_env = np.arange(N) * 6
    u = alg.selector_uniforms(N, n)
    obs, avail = rng.normal(size=(N, n, obs_dim)).astype(np.float32), sparse_avail(rng, N, n, A)
    acts = alg.predict_with_selector_envs(obs, avail, np.ones(N, bool), t_env, False, uniforms=u)
    eps = np.array([alg.selector.schedule.eval(t) for t in t_env])
    assert alg.selector.epsilon == eps[-1]
    assert np.array_equal(acts, qa.select_actions(q_of(alg.actor, N), avail, eps, u))
