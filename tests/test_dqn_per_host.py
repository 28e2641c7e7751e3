"""Prioritized replay on the host: DQN's config keys and their validation (before anything touches the device), and the
float64 sampler restatement the device tests compare against, checked on a hand-worked example."""
import numpy as np
import pytest

from per_oracle import PerTree, descend, leaf_count, weights


def _tree():
    """four slots at priorities 1, 2, 3, 4 (alpha 1): running sums 1, 3, 6, 10"""
    t = PerTree(4, alpha=1.0, eps=0.5)
    t.add(0, 4)
    assert t.update([0, 1, 2, 3], [0.5, 1.5, 2.5, 3.5]) is False
    return t


def test_tree_hand_worked():
    t = _tree()
    assert t.leaves == 4 and t.count == 4 and t.max_priority == 4.0
    assert list(t.sum) == [0, 10, 3, 7, 1, 2, 3, 4] and list(t.mn[1:]) == [1, 1, 3, 1, 2, 3, 4]
    # a later write wins; a non-finite priority is skipped; a wrapped insert enters at max_priority ** alpha
    assert t.update([2, 2, 1], [5.5, 0.5, np.nan]) is True
    assert list(t.sum[4:]) == [1, 2, 1, 4] and t.max_priority == 6.0
    t.add(0, 1)
    assert list(t.sum[4:]) == [6, 2, 1, 4] and t.sum[1] == 13 and t.mn[1] == 1


def test_sampler_hand_worked():
    t = _tree()
    # B = 2 strata of mass 5: u = 0.5 -> 2.5 (leaf 1); u = 0.25 -> 6.25 (leaf 3); u = 0.2 -> 1.0, which leaf 0's running
    # sum 1 does not exceed (leaf 1); the last stratum reaches the last stored slot (the reference's exclusive end would not)
    assert list(descend(t.sum, 4, 4, [0.5, 0.25])) == [1, 3]
    assert list(descend(t.sum, 4, 4, [0.2, 0.999999])) == [1, 3]
    # p_min = 1 / 10, max weight (0.4) ** -1 = 2.5; leaf 1: (0.8) ** -1 / 2.5 = 0.5, leaf 3: (1.6) ** -1 / 2.5 = 0.25
    np.testing.assert_allclose(weights(t.sum, t.mn, 4, 4, [1, 3], 1.0), [0.5, 0.25], rtol=1e-15)
    np.testing.assert_allclose(weights(t.sum, t.mn, 4, 4, [0, 3], 0.5), [1.0, 0.5], rtol=1e-15)


def test_sampler_clamps_to_stored_slots():
    t = PerTree(4, alpha=1.0, eps=0.5)
    t.add(0, 3)
    assert t.count == 3 and t.sum[1] == 3
    assert list(descend(t.sum, 4, 3, [0.0, 0.5, 0.999])) == [0, 1, 2]
    assert list(descend(t.sum, 4, 3, [1.0])) == [2]      # mass = total (rounding): the empty slot 3 is clamped away
    assert leaf_count(1) == 1 and leaf_count(5) == 8 and leaf_count(400000) == 2 ** 19


def test_priority_config_defaults_and_aliases():
    from xingtian_b200.algorithm.dqn import priority_config
    assert priority_config({}) == (False, 0.6, 0.4, 1e-6)
    assert priority_config({"prioritized_replay": True, "priority_alpha": 0, "PRIORITY_BETA": 1, "priority_eps": 0.01}) == \
        (True, 0.0, 1.0, 0.01)
    assert priority_config({"PRIORITIZED_REPLAY": True, "PRIORITY_ALPHA": 0.7, "priority_alpha": 0.1})[1] == 0.7


@pytest.mark.parametrize("bad", [dict(PRIORITY_ALPHA=-0.1), dict(priority_alpha=float("inf")), dict(PRIORITY_BETA=0),
                                 dict(priority_beta=-1.0), dict(PRIORITY_EPS=0.0), dict(priority_eps=float("nan")),
                                 dict(prioritized_replay=1), dict(prioritized_replay="yes"), dict(PRIORITY_BETA=True),
                                 dict(PRIORITY_ALPHA="0.5")])
def test_dqn_rejects_bad_priority_config_before_the_device(bad):
    """DQN raises while reading its config, before the models or the replay ring are built (no GPU needed)"""
    from xingtian_b200.algorithm.dqn import DQN
    cfg = dict(instance_num=1, agent_num=1, prioritized_replay=True)
    cfg.update(bad)
    info = {"actor": {"model_name": "DqnMlp", "state_dim": [4], "action_dim": 2, "model_config": {}}}
    with pytest.raises(ValueError):
        DQN(info, cfg)
