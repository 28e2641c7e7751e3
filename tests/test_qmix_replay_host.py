"""CPU tier of QMixAlg's device replay (DEVICE_REPLAY): the config check, the host bookkeeping against ReplayBuffer, the
packed episode row against what EpisodeBatch.update stores, and the refusals at prepare_data.  Nothing here touches
CUDA: the native ring is replaced by a recorder of the rows it would store."""
import numpy as np
import pytest

import qmix_alg_scenario as sc


def _scheme_parts():
    from xingtian_b200.algorithm.qmix import OneHot
    n, A, T = sc.N_AGENTS, sc.N_ACTIONS, sc.LIMIT + 1
    scheme = {
        "state": {"vshape": sc.STATE},
        "obs": {"vshape": sc.OBS, "group": "agents"},
        "actions": {"vshape": (1,), "group": "agents", "dtype": np.int64},
        "avail_actions": {"vshape": (A,), "group": "agents", "dtype": np.int32},
        "reward": {"vshape": (1,)},
        "terminated": {"vshape": (1,), "dtype": np.uint8},
        "actions_onehot": {"vshape": (A,), "dtype": np.float32, "group": "agents"},
    }
    return scheme, {"agents": n}, T, {"actions": ("actions_onehot", [OneHot(out_dim=A)])}


class _RecordingRing(object):
    """DeviceEpisodeReplay's native side replaced: _store records (slot, row)."""

    def _create(self):
        self.stored = []

    def _store(self, slot, row):
        self.stored.append((slot, row.copy()))


def _recording_alg(monkeypatch, **extra):
    from xingtian_b200.algorithm import qmix
    from xingtian_b200.registry import Registers

    class QmixReplayRecordingModel(sc.RecordingActor):
        pass

    Registers.model(QmixReplayRecordingModel)
    monkeypatch.setattr(qmix, "DeviceEpisodeReplay", type("Rec", (_RecordingRing, qmix.DeviceEpisodeReplay), {}))
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixReplayRecordingModel"
    alg_config.update(extra)
    return qmix.QMixAlg(model_info, alg_config)


@pytest.mark.parametrize("key,value", [("DEVICE_REPLAY", 1), ("DEVICE_REPLAY", "True"), ("device_replay", None),
                                       ("device_replay", 0.0)])
def test_device_replay_must_be_a_bool_and_is_checked_before_cuda(key, value):
    """The model (the first thing that touches CUDA) is never built: the check comes before it."""
    from xingtian_b200.algorithm.qmix import QMixAlg
    from xingtian_b200.registry import Registers

    class QmixNeverBuiltModel(sc.RecordingActor):
        def __init__(self, model_info=None):
            raise AssertionError("the model was built before the config check")

    Registers.model(QmixNeverBuiltModel)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixNeverBuiltModel"
    alg_config[key] = value
    with pytest.raises(ValueError, match=key):
        QMixAlg(model_info, alg_config)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixNeverBuiltModel"
    alg_config.update(DEVICE_REPLAY=True, device_replay=False)
    with pytest.raises(ValueError, match="disagree"):
        QMixAlg(model_info, alg_config)


def test_lower_case_key_and_explore_scene(monkeypatch):
    alg = _recording_alg(monkeypatch, device_replay=True)
    assert alg.device_replay and alg.buffer.stored == []
    from xingtian_b200.algorithm import qmix
    from xingtian_b200.registry import Registers

    class QmixExploreModel(sc.RecordingActor):
        pass

    Registers.model(QmixExploreModel)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixExploreModel"
    alg_config["DEVICE_REPLAY"] = True
    explore = qmix.QMixAlg(model_info, alg_config, scene="explore")
    assert not explore.device_replay and isinstance(explore.buffer, qmix.ReplayBuffer)


@pytest.mark.parametrize("batches", [[1] * 23, [1, 2, 3, 4, 5, 1, 7, 1, 2, 6]])
def test_ring_bookkeeping_and_draws_match_replay_buffer(batches):
    from xingtian_b200.algorithm.qmix import EpisodeBatch, EpisodeRing, ReplayBuffer
    scheme, groups, T, pre = _scheme_parts()
    size, bs = 6, 4
    host, ring = ReplayBuffer(scheme, groups, size, T, preprocess=pre), EpisodeRing(size)
    k = 0
    for step, nb in enumerate(batches):
        ep = EpisodeBatch(scheme, groups, nb, T, preprocess=pre)
        ep.data["state"][:] = np.arange(k, k + nb, dtype=np.float32)[:, None, None]   # episode number as a marker
        slots = ring.insert(nb)
        host.insert_episode_batch(ep)
        assert (ring.buffer_index, ring.episodes_in_buffer) == (host.buffer_index, host.episodes_in_buffer)
        assert [host.data["state"][s, 0, 0] for s in slots[-size:]] == list(np.arange(k, k + nb, dtype=np.float32)[-size:])
        k += nb
        assert ring.can_sample(bs) == host.can_sample(bs)
        if not host.can_sample(bs):
            with pytest.raises(ValueError):
                ring.sample(bs)
            continue
        np.random.seed(step)
        ids = ring.sample(bs)
        after = np.random.get_state()[1].copy()
        np.random.seed(step)
        batch = host.sample(bs)
        assert np.array_equal(np.random.get_state()[1], after)
        assert np.array_equal(batch["state"], host.data["state"][ids])
        if host.episodes_in_buffer == bs:
            assert ids.tolist() == list(range(bs))


def _episode_dict(i, onehot_order=None):
    """sc.episode(i) with every field in another dtype than the scheme's (the packer converts), and optionally a caller
    actions_onehot before or after actions."""
    d, m = sc.episode(i)
    rng = np.random.default_rng(i)
    out = dict(state=d["state"].astype(np.float64) + 1e-9, obs=d["obs"].astype(np.float64).tolist(),
               actions=d["actions"].astype(np.float64), avail_actions=d["avail_actions"].astype(np.float32),
               reward=d["reward"].astype(np.float64) / 3, terminated=d["terminated"].astype(bool), filled=d["filled"].astype(np.int32))
    if onehot_order is not None:
        oh = rng.random((sc.LIMIT + 1, sc.N_AGENTS, sc.N_ACTIONS)) / 7
        items = list(out.items())
        pos = [k for k, _ in items].index("actions") + (1 if onehot_order == "after" else 0)
        items.insert(pos, ("actions_onehot", oh))
        out = dict(items)
    return out


@pytest.mark.parametrize("onehot_order", [None, "before", "after"])
def test_packed_row_is_what_the_host_ring_stores(onehot_order):
    from xingtian_b200.algorithm.qmix import EpisodeBatch, EpisodeRowPacker, ReplayBuffer
    scheme, groups, T, pre = _scheme_parts()
    host = ReplayBuffer(scheme, groups, 3, T, preprocess=pre)
    packer = EpisodeRowPacker(scheme, groups, T, pre)
    for i in range(5):
        data = _episode_dict(i, onehot_order)
        host.insert_episode_batch(EpisodeBatch(scheme, groups, 1, T, data=dict(data)))
        slot = (host.buffer_index - 1) % 3
        row = packer.pack(dict(data))
        assert row.dtype == np.uint8 and row.size == packer.row_bytes and packer.row_bytes % 16 == 0
        got = packer.fields(row)
        for key, dt in (("state", np.float32), ("obs", np.float32), ("actions", np.int32), ("actions_onehot", np.float32),
                        ("avail_actions", np.int32), ("reward", np.float32), ("terminated", np.uint8), ("filled", np.int64)):
            want = host.data[key][slot]
            assert got[key].dtype == dt
            assert np.array_equal(got[key].reshape(want.shape), want.astype(dt)), key
        if onehot_order == "after":      # the caller's one-hot wins, rounded once to float32
            assert not np.array_equal(got["actions_onehot"], np.eye(sc.N_ACTIONS, dtype=np.float32)[got["actions"][..., 0]])
        else:
            assert np.array_equal(got["actions_onehot"], np.eye(sc.N_ACTIONS, dtype=np.float32)[got["actions"][..., 0]])


def test_missing_field_is_refused():
    from xingtian_b200.algorithm.qmix import EpisodeRowPacker
    scheme, groups, T, pre = _scheme_parts()
    data = _episode_dict(0)
    del data["filled"]
    with pytest.raises(ValueError, match="filled"):
        EpisodeRowPacker(scheme, groups, T, pre).pack(data)


@pytest.mark.parametrize("case", ["action_high", "action_negative", "filled_over", "filled_negative"])
def test_bad_episodes_raise_at_prepare_data_before_anything_is_stored(monkeypatch, case):
    alg = _recording_alg(monkeypatch, DEVICE_REPLAY=True)
    d, m = sc.episode(1)
    alg.prepare_data(dict(d))
    assert len(alg.buffer.stored) == 1 and alg.buffer.episodes_in_buffer == 1
    d = {k: v.copy() for k, v in d.items()}
    if case == "action_high":
        d["actions"][sc.LIMIT - 1, 1, 0] = sc.N_ACTIONS
    elif case == "action_negative":
        d["actions"][0, 0, 0] = -1
    elif case == "filled_over":
        d["filled"][:] = 1
        d["filled"][0] = 2
    else:
        d["filled"][:] = 0
        d["filled"][3] = -1
    with pytest.raises(ValueError):
        alg.prepare_data(d)
    assert len(alg.buffer.stored) == 1 and alg.buffer.episodes_in_buffer == 1 and alg.buffer.buffer_index == 1


def test_prepare_data_draws_as_the_host_buffer(monkeypatch):
    """The device alg's ids equal the host alg's sampled rows, with the np.random stream in the same state after."""
    from xingtian_b200.algorithm.qmix import QMixAlg
    dev = _recording_alg(monkeypatch, DEVICE_REPLAY=True)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "QmixReplayRecordingModel"
    host = QMixAlg(model_info, alg_config)
    for i in range(sc.N_EPISODES):
        d, _ = sc.episode(i)
        np.random.seed(i)
        dev.prepare_data(dict(d))
        st = np.random.get_state()[1].copy()
        np.random.seed(i)
        host.prepare_data(dict(d))
        assert np.array_equal(np.random.get_state()[1], st)
        assert (dev.train_batch is None) == (host.train_batch is None)
        if dev.train_batch is not None:
            assert np.array_equal(host.buffer.data["state"][dev.train_batch], host.train_batch["state"])
        assert dev.buffer.stored[-1][0] == (host.buffer.buffer_index - 1) % alg_config["buffer_size"]
