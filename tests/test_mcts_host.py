"""CPU tier of the MuZero tree search: the float64 lock-step restatement (tests/mcts_oracle.py) driven by the stand-in
network through the agent mirror (xingtian_b200/agent/muzero.py) reproduces the reference's searches, seeded draws and
chosen actions in tests/golden/mcts.npz bit for bit; lock-stepped trees are independent; data_proc equals the
reference's; and the search predict_fn answers BatchedPredictor requests row by row."""
import os
import queue
import sys

import numpy as np
import pytest

import mcts_oracle as mo
from xingtian_b200.agent.muzero import Muzero, MuzeroAtari, search_predict_fn
from xingtian_b200.service import BatchedPredictor, make_msg

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_mcts as gm  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "mcts.npz"))


class _SearchActor(object):
    """MuzeroModel.search's interface, computed by the oracle on the stand-in network."""

    def __init__(self, A, seed=None):
        self.action_dim = A
        self.net = mo.StandIn(gm.OBS_DIM, A, seed=A if seed is None else seed)
        self.calls = []

    def search(self, obs, num_simulations, noise=None, pb_c_base=None, pb_c_init=None, discount=None, exploration_frac=None):
        self.calls.append(len(obs))
        counts, root_value, _ = mo.search(self.net.initial, self.net.recurrent, np.asarray(obs, np.float32), num_simulations,
                                          noise, pb_c_base, pb_c_init, discount, exploration_frac)
        return counts.astype(np.int32), root_value


def _agent(A, S, cls=Muzero):
    alg = type("Alg", (), {})()
    alg.actor = _SearchActor(A)
    return cls(alg=alg, agent_config={"NUM_SIMULATIONS": S})


@pytest.mark.parametrize("case", range(len(gm.CASES)), ids=[gm.case_key(*c) for c in gm.CASES])
def test_agent_on_oracle_reproduces_reference_search_bit_for_bit(case):
    A, S, explore = gm.CASES[case]
    key = gm.case_key(A, S, explore)
    agent = _agent(A, S)
    np.random.seed(gm.case_seed(case))
    for t, obs in enumerate(gm.case_obs(A, S, explore)):
        action = agent.infer_action(obs, explore)
        td = agent.transition_data
        assert action == G[key + "_action"][t]
        assert td["child_visits"] == G[key + "_child_visits"][t].tolist()
        assert td["root_value"] == G[key + "_root_value"][t]
        assert td["cur_state"] is obs
    # the visit counts themselves, and the first expansion of every search at the highest action
    counts, _, _ = mo.search(agent.alg.actor.net.initial, agent.alg.actor.net.recurrent, gm.case_obs(A, S, explore), S)
    if not explore:
        np.testing.assert_array_equal(counts, G[key + "_counts"])
    assert (G[key + "_counts"].sum(1) == S).all()
    if S == 1:
        assert (G[key + "_counts"][:, A - 1] == 1).all()


def test_lock_step_trees_are_independent():
    A, S = 6, 50
    net = mo.StandIn(gm.OBS_DIM, A, seed=3)
    obs = np.random.default_rng(0).normal(size=(5, gm.OBS_DIM)).astype(np.float32)
    noise = np.random.default_rng(1).dirichlet([0.25] * A, 5)
    counts, root_value, margin = mo.search(net.initial, net.recurrent, obs, S, noise)
    assert margin > 0
    for e in range(5):
        c1, v1, _ = mo.search(net.initial, net.recurrent, obs[e:e + 1], S, noise[e:e + 1])
        np.testing.assert_array_equal(c1[0], counts[e])
        assert v1[0] == root_value[e]


def test_infer_actions_draws_all_noise_then_all_actions():
    A, S = 6, 2
    agent = _agent(A, S)
    obs = np.random.default_rng(2).normal(size=(3, gm.OBS_DIM)).astype(np.float32)
    np.random.seed(7)
    action, child_visits, root_value = agent.infer_actions(obs, True)
    assert agent.alg.actor.calls == [3]
    np.random.seed(7)
    noise = np.stack([np.random.dirichlet([0.25] * A) for _ in range(3)])
    counts, rv, _ = mo.search(agent.alg.actor.net.initial, agent.alg.actor.net.recurrent, obs, S, noise)
    expect = [np.random.choice(A, p=c / c.sum()) for c in counts.astype(np.float64)]
    np.testing.assert_array_equal(action, expect)
    np.testing.assert_array_equal(child_visits, counts / counts.sum(1, keepdims=True))
    np.testing.assert_array_equal(root_value, rv)


def test_atari_agent_casts_frames_to_uint8():
    agent = _agent(2, 1, MuzeroAtari)
    assert agent.keep_seq_len and agent.num_simulations == 1
    state = np.array([[1.7, 300.0, -1.0, 2.0, 5.0]])
    np.random.seed(0)
    agent.infer_action(state[0], False)
    assert agent.transition_data["cur_state"].dtype == np.uint8
    np.testing.assert_array_equal(agent.transition_data["cur_state"], state[0].astype("uint8"))


@pytest.mark.parametrize("e", range(int(G["n_episodes"])))
def test_data_proc_matches_reference(e):
    agent = _agent(2, 1)
    for k in ("root_value", "reward", "done"):
        agent.trajectory[k] = G["ep%d_%s" % (e, k)].tolist()
    agent.handle_env_feedback(None, 1.0, False, {}, True)
    traj = agent.get_trajectory()
    assert [float(x) for x in traj["target_value"]] == G["ep%d_target_value" % e].tolist()


def test_search_predict_fn_scatters_rows_to_explorers():
    A, S = 6, 2
    actor = _SearchActor(A)
    actor.state_dim = [gm.OBS_DIM]
    alg = type("Alg", (), {"actor": actor})()
    req, rep = queue.Queue(), queue.Queue()
    svc = BatchedPredictor(0, alg, req, rep, predict_fn=search_predict_fn(actor, S, use_explore=True), max_wait_s=0.05)
    obs = np.random.default_rng(4).normal(size=(3, gm.OBS_DIM)).astype(np.float32)
    req.put(make_msg(obs[0], cmd="predict", explorer_id=0))       # one observation
    req.put(make_msg(obs[1:], cmd="predict", explorer_id=1))      # two stacked observations
    np.random.seed(11)
    assert svc.process_once(timeout=1.0) == 2
    assert actor.calls == [3]                                     # one search for both explorers
    np.random.seed(11)
    noise = np.stack([np.random.dirichlet([0.25] * A) for _ in range(3)])
    counts, rv, _ = mo.search(actor.net.initial, actor.net.recurrent, obs, S, noise)
    expect_a = [np.random.choice(A, p=c / c.sum()) for c in counts.astype(np.float64)]
    r0, r1 = rep.get_nowait(), rep.get_nowait()
    assert r0["ctr_info"]["explorer_id"] == 0 and r1["ctr_info"]["explorer_id"] == 1
    a0, cv0, v0 = r0["data"]
    assert a0 == expect_a[0] and v0 == rv[0]
    np.testing.assert_array_equal(cv0, counts[0] / counts[0].sum())
    a1, cv1, v1 = r1["data"]
    np.testing.assert_array_equal(a1, expect_a[1:])
    np.testing.assert_array_equal(cv1, counts[1:] / counts[1:].sum(1, keepdims=True))
    np.testing.assert_array_equal(v1, rv[1:])
