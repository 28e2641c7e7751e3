"""The MuZero tree search on the H100 (xtb_muzero_search) against the float64 lock-step restatement (tests/mcts_oracle.py)
driven by the same model's own batched inference calls: identical visit counts and root values for MuzeroMlp and
MuzeroCnn (uint8 and int8 frames) at N in {1, 7, 50} trees, S in {1, 2, 50} simulations, with and without root noise;
graph replay against eager launches; repeat calls; the seeded agent against the oracle run through the batch-1 public
calls; argument checks that launch nothing; and the BatchedPredictor answering two explorers from one search.

The oracle's UCB uses libm's log and the kernel CUDA's, which may differ in the last ulp, so every case first asserts that
each descent decision not settled by construction has a relative margin above 1e-12: a seed that fails that premise is a
bad fixture, not a pass."""
import ctypes as C
import queue

import numpy as np
import pytest
import torch

import mcts_oracle as mo
from test_gpu_kernels import one_rank_comm

pytestmark = pytest.mark.gpu

MODELS = {   # kind -> (model name, state_dim, A, model_config)
    "mlp": ("MuzeroMlp", [4], 2, {}),
    "cnn_u8": ("MuzeroCnn", [84, 84, 4], 4, dict(obs_type="uint8", reward_min=0, reward_max=50, value_min=0, value_max=500)),
    "cnn_i8": ("MuzeroCnn", [84, 84, 4], 6, dict(obs_type="int8", reward_min=-2, reward_max=2, value_min=-21, value_max=21)),
}
_cache = {}


def _model(kind, graph=True, fresh=False):
    key = (kind, graph)
    if fresh or key not in _cache:
        from xingtian_b200.registry import Registers
        torch.cuda.set_device(0)
        name, sd, A, cfg = MODELS[kind]
        mc = dict(cfg, init_seed=1, use_cuda_graph=graph, max_batch=64)
        _cache[key] = Registers.model[name]({"model_name": name, "state_dim": sd, "action_dim": A, "model_config": mc})
    return _cache[key]


def _obs(m, n, seed):
    rng = np.random.default_rng(seed)
    if len(m.state_dim) == 3:
        return rng.integers(0, 256, (n,) + tuple(m.state_dim)).astype(np.uint8)
    return rng.normal(size=(n,) + tuple(m.state_dim)).astype(np.float32)


def _batched_callbacks(m, obs):
    """initial / recurrent callbacks of the oracle on the model's batched device calls at the batch size of obs."""
    n = len(obs)
    b = m._buffers(n)
    from xingtian_b200.engine import stage_h2d
    stage_h2d(b["obs"], m._host_obs(obs), m._np_dt)

    def initial(_):
        _, policy, hidden = m.initial_inference_batch(b["obs"], n)
        return policy.cpu().numpy(), list(hidden.clone())

    def recurrent(hidden_rows, actions):
        h = torch.stack(hidden_rows).contiguous()
        a = torch.tensor(actions, dtype=torch.int32, device=m.device)
        value, reward, policy, hid = m.recurrent_inference_batch(h, a, n)
        return value.cpu().numpy(), reward.cpu().numpy(), policy.cpu().numpy(), list(hid.clone())
    return initial, recurrent


def _check_parity(m, obs, S, noise):
    counts, rv = m.search(obs, S, noise=noise)
    initial, recurrent = _batched_callbacks(m, obs)
    rc, rrv, margin = mo.search(initial, recurrent, obs, S, noise)
    assert margin > 1e-12, "bad fixture: a UCB decision within %g relative" % margin
    np.testing.assert_array_equal(counts, rc)
    assert np.all(np.abs(rv - rrv) <= 1e-12 * np.maximum(np.abs(rrv), 1e-300)), (rv, rrv)
    assert (counts.sum(1) == S).all()
    return counts, rv


@pytest.mark.parametrize("explore", [False, True], ids=["plain", "noise"])
@pytest.mark.parametrize("S", [1, 2, 50])
@pytest.mark.parametrize("n", [1, 7, 50])
@pytest.mark.parametrize("kind", list(MODELS))
def test_search_matches_oracle_on_the_models_own_inference(kind, n, S, explore):
    m = _model(kind)
    A = m.action_dim
    obs = _obs(m, n, seed=n * 7 + S)
    noise = np.random.default_rng(S + n).dirichlet([0.25] * A, n) if explore else None
    counts, _ = _check_parity(m, obs, S, noise)
    if S == 1:
        assert (counts[:, A - 1] == 1).all()       # N_p = 0: every score is 0 and the highest action is expanded first


def test_graph_replay_equals_eager_and_repeats():
    mg, me = _model("cnn_i8", graph=True), _model("cnn_i8", graph=False)
    me.set_weights(mg.get_weights())
    obs = _obs(mg, 7, seed=3)
    noise = np.random.default_rng(0).dirichlet([0.25] * 6, 7)
    from xingtian_b200 import capi
    lib = capi.lib()
    c1, v1 = mg.search(obs, 50, noise=noise)
    replays = lib.xtb_graph_replay_count()
    c2, v2 = mg.search(obs, 50, noise=noise)
    assert lib.xtb_graph_replay_count() == replays + 1
    c3, v3 = me.search(obs, 50, noise=noise)
    for c, v in ((c2, v2), (c3, v3)):
        np.testing.assert_array_equal(c, c1)
        np.testing.assert_array_equal(v, v1)


class _BatchOneActor(object):
    """The oracle through the model's public batch-1 host calls (initial_inference / recurrent_inference)."""

    def __init__(self, m):
        self.m, self.action_dim, self.margin = m, m.action_dim, float("inf")

    def search(self, obs, num_simulations, noise=None, pb_c_base=None, pb_c_init=None, discount=None, exploration_frac=None):
        def initial(o):
            out = [self.m.initial_inference(x[None]) for x in o]
            return np.stack([r.policy for r in out]), [r.hidden_state for r in out]

        def recurrent(hidden, actions):
            out = [self.m.recurrent_inference(h, a) for h, a in zip(hidden, actions)]
            return [r.value for r in out], [r.reward for r in out], np.stack([r.policy for r in out]), [r.hidden_state for r in out]
        counts, rv, margin = mo.search(initial, recurrent, obs, num_simulations, noise, pb_c_base, pb_c_init, discount,
                                       exploration_frac)
        self.margin = min(self.margin, margin)
        return counts.astype(np.int32), rv


@pytest.mark.parametrize("cls", ["Muzero", "MuzeroAtari"])
def test_seeded_agent_matches_oracle_through_batch_one_calls(cls):
    from xingtian_b200.agent import muzero as agent_mod
    m = _model("cnn_i8")
    Agent = getattr(agent_mod, cls)

    def run(actor):
        alg = type("Alg", (), {"actor": actor})()
        agent = Agent(alg=alg, agent_config={"NUM_SIMULATIONS": 50})
        np.random.seed(21)
        out = []
        for t, obs in enumerate(_obs(m, 4, seed=9)):
            out.append((agent.infer_action(obs, t % 2 == 0), agent.transition_data["child_visits"], agent.transition_data["root_value"]))
        return out
    ref_actor = _BatchOneActor(m)
    ref = run(ref_actor)
    assert ref_actor.margin > 1e-12, "bad fixture"
    got = run(m)
    assert [g[0] for g in got] == [r[0] for r in ref]
    assert [g[1] for g in got] == [r[1] for r in ref]
    for g, r in zip(got, ref):
        assert abs(g[2] - r[2]) <= 1e-12 * abs(r[2])


def test_argument_checks_launch_nothing():
    from xingtian_b200 import capi
    from xingtian_b200.engine import stream_ptr
    lib = capi.lib()
    m = _model("mlp")
    n = 4
    obs = torch.zeros(70, 4, device=m.device)
    counts = torch.zeros(70, 2, dtype=torch.int32, device=m.device)
    rv = torch.zeros(70, dtype=torch.float64, device=m.device)
    tree = C.c_void_p()
    capi.check(lib.xtb_muzero_tree_create(m.handle, 70, 8, C.byref(tree)))     # more trees than the model's max_batch 64
    try:
        def call(mz=m.handle, tr=tree, o=obs.data_ptr(), n=n, S=8, base=19652.0, c=counts.data_ptr(), v=rv.data_ptr()):
            return lib.xtb_muzero_search(mz, tr, o, n, S, None, base, 1.25, 0.997, 0.25, c, v, 1, stream_ptr())
        assert call() == 0
        torch.cuda.synchronize()
        before = lib.xtb_launch_count()
        for kw in (dict(mz=None), dict(tr=None), dict(o=None), dict(c=None), dict(v=None), dict(n=0), dict(n=65), dict(n=71),
                   dict(S=0), dict(S=9), dict(base=0.0), dict(base=-1.0), dict(base=float("inf")), dict(base=float("nan"))):
            assert call(**kw) == -1, kw
        with one_rank_comm():
            assert call() == -3 and b"data-parallel" in lib.xtb_last_error()
        assert lib.xtb_launch_count() == before
        assert lib.xtb_muzero_tree_create(m.handle, 0, 8, C.byref(C.c_void_p())) == -1
        assert lib.xtb_muzero_tree_create(m.handle, 4, 0, C.byref(C.c_void_p())) == -1
        assert lib.xtb_muzero_tree_create(None, 4, 8, C.byref(C.c_void_p())) == -1
    finally:
        lib.xtb_muzero_tree_destroy(tree)


def test_tree_scratch_grows_only():
    m = _model("mlp", fresh=True)
    obs = _obs(m, 7, seed=1)
    m.search(obs[:3], 2)
    assert m._tree_size == (3, 2)
    tree = m._tree.value
    m.search(obs[:2], 1)
    assert m._tree_size == (3, 2) and m._tree.value == tree
    _check_parity(m, obs, 5, None)
    assert m._tree_size == (7, 5)


def test_batched_predictor_answers_two_explorers_from_one_search():
    from xingtian_b200.agent.muzero import search_predict_fn
    from xingtian_b200.service import BatchedPredictor, make_msg
    m = _model("cnn_u8")
    calls = []
    fn = search_predict_fn(m, 50, use_explore=True)

    def counted(batch):
        calls.append(len(batch))
        return fn(batch)
    alg = type("Alg", (), {"actor": m})()
    req, rep = queue.Queue(), queue.Queue()
    svc = BatchedPredictor(0, alg, req, rep, predict_fn=counted, max_wait_s=0.05)
    obs = _obs(m, 3, seed=5)
    req.put(make_msg(obs[0], cmd="predict", explorer_id=0))
    req.put(make_msg(obs[1:], cmd="predict", explorer_id=1))
    np.random.seed(4)
    assert svc.process_once(timeout=1.0) == 2
    assert calls == [3]
    np.random.seed(4)
    action, child_visits, root_value = fn(obs)
    r0, r1 = rep.get_nowait(), rep.get_nowait()
    assert r0["ctr_info"]["explorer_id"] == 0 and r1["ctr_info"]["explorer_id"] == 1
    assert r0["data"][0] == action[0] and r0["data"][2] == root_value[0]
    np.testing.assert_array_equal(r0["data"][1], child_visits[0])
    np.testing.assert_array_equal(r1["data"][0], action[1:])
    np.testing.assert_array_equal(r1["data"][1], child_visits[1:])
    np.testing.assert_array_equal(r1["data"][2], root_value[1:])
