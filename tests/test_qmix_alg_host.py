"""CPU tier: QMixAlg's host side against tests/golden/qmix.npz, which the reference's own QMixAlg, episode buffer and
transforms produced in the same seeded session (tests/qmix_alg_scenario.py): the sampled episode ids, every array handed
to the model's train, the epsilon schedule, the selected actions and the target-sync episodes, bit for bit."""
import os

import numpy as np
import pytest

import qmix_alg_scenario as sc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qmix.npz")


@pytest.fixture(scope="module")
def session():
    from xingtian_b200.algorithm.qmix import EpisodeBatch, QMixAlg
    from xingtian_b200.registry import Registers

    class QmixRecordingModel(sc.RecordingActor):
        pass

    Registers.model(QmixRecordingModel)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixRecordingModel"
    alg = QMixAlg(model_info, alg_config)
    out = sc.drive(alg, lambda a: EpisodeBatch(a.scheme, a.groups, 1, sc.LIMIT + 1, preprocess=a.preprocess))
    out["model_obs_shape"] = np.array(model_info["actor"]["model_config"]["obs_shape"])
    out["scene"] = np.array(model_info["actor"]["scene"])
    return out, alg


def test_session_matches_the_reference_bit_for_bit(session):
    out, _ = session
    with np.load(GOLDEN) as g:
        gold = {k: g[k] for k in g.files}
    assert sorted(out) == sorted(gold)
    for k in sorted(gold):
        assert out[k].dtype == gold[k].dtype, (k, out[k].dtype, gold[k].dtype)
        assert out[k].shape == gold[k].shape, (k, out[k].shape, gold[k].shape)
        assert np.array_equal(out[k], gold[k], equal_nan=out[k].dtype.kind == "f"), k


def test_mask_and_target_sync_rules(session):
    out, alg = session
    for k in range(int(out["n_trained"])):
        term, mask = out["train%d_terminated" % k], out["train%d_mask" % k]
        # mask = filled[:, :-1] with mask[:, 1:] *= 1 - terminated[:, :-1]: nothing after a terminal step counts
        assert np.all(mask[:, 1:][term[:, :-1] == 1] == 0)
    # the first train syncs the targets, then every target_update_interval episodes
    assert out["synced_after_train"].tolist() == [1, 4, 7]
    assert alg.last_target_update_episode == 10


def test_train_ready_calls_the_dummy_model_until_a_batch_can_be_drawn():
    from xingtian_b200.algorithm.qmix import QMixAlg
    from xingtian_b200.registry import Registers

    class QmixIdleModel(sc.RecordingActor):
        pass

    Registers.model(QmixIdleModel)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixIdleModel"
    alg = QMixAlg(model_info, alg_config)
    calls = []
    assert alg.train_ready(0, dist_dummy_model=lambda: calls.append(1)) is False and calls == [1]
    with pytest.raises(KeyError):
        alg.train_ready(0)
    for i in range(alg_config["batch_size"]):
        alg.prepare_data(sc.episode(i)[0])
    assert alg.train_ready(4) is True
    assert np.isnan(QMixAlg.train(type("A", (), {"train_batch": None})()))
