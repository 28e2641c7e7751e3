"""CPU tier: DQNInfoFlowAlg's host side against the golden recorded from the reference's own algorithm
(tests/golden/infoflow.npz), the float64 restatement's targets, and the argument checks that run before any device
allocation."""
import os

import numpy as np
import pytest

import infoflow_alg_scenario as sc
import infoflow_oracle as io

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "infoflow.npz")


class _Actor(object):
    """Stand-in for DqnInfoFlowModel: records the packed minibatches and the target syncs."""
    rec = None

    def __init__(self, model_info):
        self.vocab_size = model_info["vocab_size"]

    def train_transitions(self, batch, gamma):
        _Actor.rec.trains.append((batch, gamma))
        return 0.0

    def get_weights(self):
        return ["weights"]

    def set_weights(self, weights):
        _Actor.rec.syncs.append(len(_Actor.rec.trains))


@pytest.fixture
def alg(monkeypatch):
    from xingtian_b200.algorithm.dqn_infoflow import DQNInfoFlowAlg
    from xingtian_b200.registry import Registers
    monkeypatch.setitem(Registers.model._dict, "RecordingInfoflowActor", _Actor)
    _Actor.rec = sc.Recorder()
    model_info, alg_config = sc.configs()
    return DQNInfoFlowAlg(model_info, alg_config)


def test_host_side_reproduces_the_reference_golden(alg):
    g = np.load(GOLDEN)
    out = sc.drive(alg, _Actor.rec)
    assert out["n_trained"] == int(g["n_trained"])
    np.testing.assert_array_equal(out["synced_after_train"], g["synced_after_train"])
    np.testing.assert_array_equal(np.stack(out["py_state"]), g["py_state"])
    np.testing.assert_array_equal(np.stack(out["np_key"]), g["np_key"])
    np.testing.assert_array_equal(out["np_pos"], g["np_pos"])
    for i, (b, gamma) in enumerate(_Actor.rec.trains):
        assert gamma == sc.GAMMA and int(g["t%d_batch_size" % i]) == sc.BATCH
        for mine, ref in (("user", "user_input"), ("click", "history_click"), ("noclick", "history_no_click"), ("item", "item_input")):
            assert b[mine].dtype == np.int32
            np.testing.assert_array_equal(b[mine], g["t%d_%s" % (i, ref)])
        counts = np.diff(b["cand_off"])
        assert b["cand_off"][0] == 0 and counts.min() >= 1
        for mine, ref in (("next_user", "user_input"), ("next_click", "history_click"), ("next_noclick", "history_no_click")):
            np.testing.assert_array_equal(np.repeat(b[mine], counts, axis=0), g["t%d_next_%s" % (i, ref)])
        np.testing.assert_array_equal(b["cand_item"], g["t%d_next_item_input" % i])
        # the float64 restatement's targets from the recorded Q values reproduce the reference's, bit for bit
        t = io.td_targets(g["t%d_next_q" % i], b["cand_off"], b["reward"], b["done"], gamma)
        np.testing.assert_array_equal(t, g["t%d_target" % i])
        assert b["reward"].dtype == np.float64


def _data(n=2, **over):
    rng = np.random.default_rng(0)
    d = sc.transitions(rng, 0, n)
    for k, v in over.items():
        d[k] = v
    return d


def test_prepare_data_rejects_bad_transitions_before_the_device(alg):
    bad_id = _data()
    bad_id["cur_state"][0]["user"] = [0, sc.VOCAB, 1]
    neg = _data()
    neg["next_state"][1]["candidate_items"] = [[-1, 2]]
    short = _data()
    short["cur_state"][1]["clicked_items"] = short["cur_state"][1]["clicked_items"][:-1]
    empty = _data(done=[False, False])
    empty["next_state"][0]["candidate_items"] = []
    for d in (bad_id, neg, short, empty):
        with pytest.raises(ValueError):
            alg.prepare_data(d)
    assert alg.buff.size() == 0
    done_empty = _data(done=[True, True])
    done_empty["next_state"][0]["candidate_items"] = []
    alg.prepare_data(done_empty)          # a done transition needs no candidates
    assert alg.buff.size() == 2
    floats = _data()
    floats["action"][0] = [3.7, 0.2]      # truncated toward zero by the int32 cast
    alg.prepare_data(floats)


def test_train_with_too_few_transitions_raises_index_error(alg):
    alg.prepare_data(_data(3))
    with pytest.raises(IndexError):
        alg.train(episode_num=1)
    assert _Actor.rec.trains == []


def test_train_ready_needs_the_dummy_model(alg):
    alg.learning_starts = 5
    with pytest.raises(KeyError):
        alg.train_ready(1)
    called = []
    assert alg.train_ready(1, dist_dummy_model=lambda: called.append(1)) is False and called == [1]
    assert alg.train_ready(5) is True


def test_model_rejects_bad_config_before_the_device(tmp_path, monkeypatch):
    from xingtian_b200.model import dqn_infoflow as m
    import xingtian_b200.model.base as base
    monkeypatch.setattr(base, "require_cuda", lambda: (_ for _ in ()).throw(AssertionError("reached the device")))
    path = tmp_path / "emb.csv"
    np.savetxt(path, np.zeros((10, 4)), delimiter=",")
    info = dict(state_dim=[1], action_dim=1, vocab_size=10, emb_dim=4, user_dim=1, item_dim=1, input_type="int32",
                embeddings=str(path), last_activate="hard_sigmoid")
    with pytest.raises(KeyError):
        m.DqnInfoFlowModel(info)
    with pytest.raises(ValueError):
        m.DqnInfoFlowModel(dict(info, last_activate="linear", emb_dim=138))
    with pytest.raises(ValueError):
        m.ids_int32([[0, 10]], 10, "user_input")
    np.testing.assert_array_equal(m.ids_int32(np.array([2.9, 0.5]), 10, "x"), [2, 0])
