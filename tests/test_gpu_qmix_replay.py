"""GPU tier of QMixAlg's and SCCAlg's device replay (DEVICE_REPLAY): the gathered batch against the reference's own
session (tests/golden/qmix.npz) and against the host replay's batch bit for bit, the training steps against the host
replay's, graph replay against eager launches, and the refusals."""
import contextlib
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

import qmix_alg_scenario as sc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qmix.npz")
NAMES = ("trajectories", "obs_len", "avail", "actions", "cur_stats", "target_stats", "rewards", "terminated", "mask")
H, E, HE, U = 32, 8, 16, 16


@contextlib.contextmanager
def one_rank_comm():
    """A one-rank NCCL communicator installed for the duration: the library runs its data-parallel paths on one GPU"""
    from xingtian_b200 import capi, engine
    lib = capi.lib()
    path = engine._nccl_path()
    path = path.encode() if path else None
    ident = (C.c_ubyte * 128)()
    capi.check(lib.xtb_comm_unique_id(path, ident))
    h = C.c_void_p()
    capi.check(lib.xtb_comm_create(path, ident, 0, 1, C.byref(h)))
    capi.check(lib.xtb_set_grad_comm(h))
    try:
        yield
    finally:
        capi.check(lib.xtb_set_grad_comm(None))
        lib.xtb_comm_destroy(h)


def gathered_args(replay, ids, raw_obs=False):
    """The gather of `ids` as the host path's train arguments (NAMES order; the raw obs second when raw_obs), on the host."""
    b = replay.gather(ids)
    h = {k: v.cpu().numpy() for k, v in b.items() if k != "batch"}
    max_t = int(h["max_t"][0])
    assert np.all(h["seq_len"] == max_t)
    args = [h["obs"], h["seq_len"], h["avail"], h["actions"][..., None], h["state"], h["next_state"], h["reward"][..., None],
            h["terminated"][..., None], h["mask"][..., None]]
    if raw_obs:
        args.insert(1, h["raw_obs"])
    return args, max_t


def assert_same_batch(dev_args, host_args, what):
    """Device float32 / int32 arrays equal the host arrays exactly: the host values are representable in the device dtype
    and the device values are those values."""
    assert len(dev_args) == len(host_args)
    for k, (d, h) in enumerate(zip(dev_args, host_args)):
        h = np.asarray(h)
        assert d.size == h.size, (what, k, d.shape, h.shape)
        hd = h.astype(d.dtype).reshape(d.shape)
        assert np.array_equal(hd.astype(h.dtype).reshape(h.shape), h), (what, k, "host values not representable")
        assert np.array_equal(d, hd), (what, k, np.argwhere(d != hd)[:5])


class GatherActor(sc.RecordingActor):
    """The scenario's actor on the device replay: train_replay gathers the batch and records it as train's arguments."""

    def train_replay(self, replay, ids):
        args, max_t = gathered_args(replay, ids)
        self.trained.append(args)
        return float(len(self.trained)), max_t


def scenario_alg(device_replay, **over):
    from xingtian_b200.algorithm.qmix import QMixAlg
    from xingtian_b200.registry import Registers

    class QmixGatherModel(GatherActor):
        pass

    class QmixHostRecordingModel(sc.RecordingActor):
        pass

    Registers.model(QmixGatherModel)
    Registers.model(QmixHostRecordingModel)
    model_info, alg_config = sc.configs()
    alg_config.update(over, DEVICE_REPLAY=device_replay)
    model_info["actor"]["model_name"] = "QmixGatherModel" if device_replay else "QmixHostRecordingModel"
    return QMixAlg(model_info, alg_config)


def new_batch(alg):
    from xingtian_b200.algorithm.qmix import EpisodeBatch
    return EpisodeBatch(alg.scheme, alg.groups, 1, sc.LIMIT + 1, preprocess=alg.preprocess)


def test_reference_session_bit_for_bit():
    """The reference's seeded session, every batch gathered on the device: all train*_ arrays, and the draws, actions,
    epsilons, ready flags and syncs, equal tests/golden/qmix.npz."""
    torch.cuda.set_device(0)
    alg = scenario_alg(True)
    assert alg.device_replay
    out = sc.drive(alg, new_batch)
    with np.load(GOLDEN) as g:
        gold = {k: g[k] for k in g.files}
    n_trained = int(gold["n_trained"])
    assert n_trained > 0 and int(out["n_trained"]) == n_trained
    for k in range(n_trained):
        assert_same_batch([out["train%d_%s" % (k, name)] for name in NAMES], [gold["train%d_%s" % (k, name)] for name in NAMES],
                          "train %d" % k)
    for key in sorted(gold):
        if key.startswith("train") or key in ("model_obs_shape", "scene"):
            continue
        assert np.array_equal(out[key], gold[key], equal_nan=out[key].dtype.kind == "f"), key


@pytest.mark.parametrize("last_action,agent_id,buffer_size", [(True, True, 6), (True, False, 6), (False, True, 6),
                                                              (False, False, 6), (True, True, 4)])
def test_gathered_batch_equals_host_batch(last_action, agent_id, buffer_size):
    """Both build_inputs switches, and buffer_size == batch_size (no draw at all): the session on the host replay and on
    the device replay hands the model the same arrays."""
    torch.cuda.set_device(0)
    over = dict(obs_last_action=last_action, obs_agent_id=agent_id, buffer_size=buffer_size)
    host, dev = scenario_alg(False, **over), scenario_alg(True, **over)
    oh, od = sc.drive(host, new_batch), sc.drive(dev, new_batch)
    assert int(oh["n_trained"]) == int(od["n_trained"]) > 0
    assert int(od["n_sampled"]) == (0 if buffer_size == 4 else int(oh["n_sampled"]))
    for k in range(int(oh["n_trained"])):
        assert_same_batch([od["train%d_%s" % (k, name)] for name in NAMES], [oh["train%d_%s" % (k, name)] for name in NAMES],
                          "train %d" % k)
    for key in ("acted", "epsilon", "ready", "synced_after_train", "losses"):
        assert np.array_equal(oh[key], od[key], equal_nan=oh[key].dtype.kind == "f"), key


# ---- the real models ------------------------------------------------------------------------------------------------
N, A, OBS, SD, L, B, BUF = 3, 5, 6, 7, 10, 4, 6


def real_alg(kind, device_replay, seed=3, use_graph=True, last_action=True, agent_id=True, multi=True):
    from xingtian_b200.algorithm.qmix import QMixAlg
    from xingtian_b200.algorithm.scc import SCCAlg
    env_attr = dict(n_agents=N, n_actions=A, state_shape=SD, obs_shape=OBS, episode_limit=L)
    alg_config = dict(batch_size=B, buffer_size=BUF, epsilon_anneal_time=40, epsilon_finish=0.05, epsilon_start=1.0,
                      obs_agent_id=agent_id, obs_last_action=last_action, target_update_interval=3, env_attr=env_attr,
                      instance_num=1, agent_num=1, DEVICE_REPLAY=device_replay)
    mc = dict(gamma=0.99, n_agents=N, rnn_hidden_dim=H, episode_limit=L, n_actions=A, batch_size=B, state_shape=[SD],
              use_double_q=True, init_seed=seed, use_cuda_graph=use_graph)
    if kind == "qmix":
        mc.update(lr=0.0005, grad_norm_clip=10, mixing_embed_dim=E, hypernet_embed=HE, hypernet_layers=2)
        return QMixAlg({"actor": {"model_name": "QMixModel", "model_config": mc}}, alg_config)
    mc.update(mixer_grad_norm_clip=5, actor_grad_norm_clip=5, a_lr=0.0005, c_lr=0.0005, dense_unit_number=U,
              enable_critic_multi_channel=multi, channel_merge="concat", mc_sample_times=2, map_name="x")
    return SCCAlg({"actor": {"model_name": "SCCModel", "model_config": mc}}, alg_config)


def episode_stream(count, seed=5):
    """Episodes of 1 to L + 1 steps (both ends included), every other one terminated."""
    rng = np.random.default_rng(seed)
    T = L + 1
    lengths = [1, T] + [int(x) for x in rng.integers(1, T + 1, size=count - 2)]
    for i, m in enumerate(lengths):
        d = dict(state=np.zeros((T, SD), np.float32), obs=np.zeros((T, N, OBS), np.float32), actions=np.zeros((T, N, 1), np.int64),
                 avail_actions=np.zeros((T, N, A), np.int32), reward=np.zeros((T, 1), np.float32),
                 terminated=np.zeros((T, 1), np.uint8), filled=np.zeros((T, 1), np.int64))
        d["state"][:m] = rng.normal(size=(m, SD))
        d["obs"][:m] = rng.normal(size=(m, N, OBS))
        d["avail_actions"][:m] = (rng.random((m, N, A)) < 0.6)
        d["avail_actions"][:m, :, 0] = 1
        d["actions"][:m, :, 0] = rng.integers(0, A, size=(m, N))
        d["reward"][:m, 0] = rng.normal(size=m)
        d["terminated"][m - 1, 0] = i % 2
        d["filled"][:m] = 1
        yield d


def record_host_train(alg):
    """Record the arguments the host path hands the model's train."""
    model, calls = alg.actor, []
    orig = model.train

    def train(*args):
        calls.append([np.array(a) for a in args])
        return orig(*args)

    model.train = train
    return calls


def device_batch(model, raw_obs):
    b = {k: v.cpu().numpy() for k, v in model._train_buffers().items()}
    args = [b["obs"], b["seq_len"]] + ([] if raw_obs else [b["avail"]]) + [b["actions"][..., None]]
    args += [] if raw_obs else [b["state"], b["next_state"]]
    args += [b["reward"][..., None], b["terminated"][..., None], b["mask"][..., None]]
    if raw_obs:
        args.insert(1, b["raw_obs"][..., :model.o_shape])
    return args


def host_batch(args, raw_obs):
    """The host arguments the device buffers hold (SCC's model buffers have no avail or states)."""
    return [a for i, a in enumerate(args) if not (raw_obs and i in (3, 5, 6))]   # avail, cur_stats, target_stats


def run_pair(kind, count=12, **kw):
    """Host and device replay algs with the same init_seed on the same episodes and draws -> (host, device, losses)."""
    torch.cuda.set_device(0)
    host, dev = real_alg(kind, False, **kw), real_alg(kind, True, **kw)
    assert dev.device_replay and not host.device_replay
    calls = record_host_train(host)
    raw = kind == "scc"
    losses = []
    for i, d in enumerate(episode_stream(count)):
        for alg in (host, dev):
            np.random.seed(1000 + i)
            alg.prepare_data({k: v.copy() for k, v in d.items()})
        assert (host.train_batch is None) == (dev.train_batch is None)
        if dev.train_batch is None:
            continue
        assert np.array_equal(host.train_batch["state"], host.buffer.data["state"][dev.train_batch])
        out = []
        for alg in (host, dev):
            random.seed(2000 + i)
            out.append(alg.train(episode_num=i + 1))
        losses.append(out)
        assert_same_batch(device_batch(dev.actor, raw), host_batch(calls[-1], raw), "step %d" % len(losses))
    assert dev.buffer.episodes_in_buffer == BUF and count > BUF + 2 and len(losses) >= 5
    return host, dev, np.array(losses)


def check_pair(host, dev, losses):
    assert losses[0, 0] == losses[0, 1]
    np.testing.assert_allclose(losses[:, 1], losses[:, 0], rtol=1e-5, atol=1e-5)
    for a, c in ((dev.actor.params, host.actor.params), (dev.actor.target, host.actor.target), (dev.actor.explore, host.actor.explore)):
        torch.testing.assert_close(a, c, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("switches", [(True, True), (False, False)], ids=["inputs_full", "obs_only"])
def test_qmix_device_replay_trains_as_host_replay(switches):
    check_pair(*run_pair("qmix", last_action=switches[0], agent_id=switches[1]))


@pytest.mark.parametrize("multi", [True, False], ids=["multi_channel", "single_channel"])
def test_scc_device_replay_trains_as_host_replay(multi):
    host, dev, losses = run_pair("scc", multi=multi)
    check_pair(host, dev, losses)
    assert dev.actor.mixer_loss == pytest.approx(host.actor.mixer_loss, rel=1e-5, abs=1e-5)


def test_graph_replay_matches_eager_and_one_capture_serves_the_ring():
    """A graph and an eager device-replay alg on the same stream: the same first loss, later ones to rounding, and no new
    capture after the first train() while max_ep_t varies and the ring fills and wraps."""
    from xingtian_b200 import capi
    torch.cuda.set_device(0)
    g, e = real_alg("qmix", True, use_graph=True), real_alg("qmix", True, use_graph=False)
    lib = capi.lib()
    losses, captures, max_ts = [], None, set()
    for i, d in enumerate(episode_stream(14, seed=9)):
        for alg in (g, e):
            np.random.seed(3000 + i)
            alg.prepare_data({k: v.copy() for k, v in d.items()})
        if g.train_batch is None:
            continue
        max_ts.add(int(g.buffer.gather(g.train_batch)["max_t"].cpu()[0]))
        losses.append((g.train(episode_num=i + 1), e.train(episode_num=i + 1)))
        if captures is None:
            captures = lib.xtb_graph_capture_count()
        assert lib.xtb_graph_capture_count() == captures
    losses = np.array(losses)
    assert len(losses) >= 8 and len(max_ts) >= 2
    assert losses[0, 0] == losses[0, 1]
    np.testing.assert_allclose(losses[:, 0], losses[:, 1], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(g.actor.params, e.actor.params, rtol=1e-5, atol=1e-7)


def test_invalid_arguments_launch_nothing_and_a_communicator_is_refused():
    from xingtian_b200 import capi
    from xingtian_b200.algorithm.qmix import DeviceEpisodeReplay, EpisodeBatch
    from xingtian_b200.engine import _ptr, stream_ptr
    torch.cuda.set_device(0)
    lib = capi.lib()
    algs = {kind: real_alg(kind, True) for kind in ("qmix", "scc")}
    stream = list(episode_stream(B))
    for alg in algs.values():
        for d in stream:
            alg.prepare_data(d)
    alg = algs["qmix"]
    rep, model = alg.buffer, alg.actor
    assert rep.episodes_in_buffer == B and alg.train_batch is not None
    row = rep.packer.pack(stream[0])
    b = rep.buffers(B)
    model._train_buffers()
    out = model._replay_out(1)
    launches = lib.xtb_launch_count()

    def gather(ids, n=None):
        ids = np.ascontiguousarray(ids, np.int32)
        return lib.xtb_episode_replay_gather(rep.handle, len(ids) if n is None else n, ids.ctypes.data, C.byref(b["batch"]),
                                             _ptr(b["max_t"]), stream_ptr())

    def train(ids, replay=rep):
        ids = np.ascontiguousarray(ids, np.int32)
        mb = model._train_buffers()
        bt = capi.QmixBatch()
        for k in ("obs", "seq_len", "avail", "actions", "state", "next_state", "reward", "terminated", "mask"):
            setattr(bt, k, mb[k].data_ptr())
        return lib.xtb_qmix_replay_train(replay.handle, model.handle, model.opt.handle, _ptr(model.target), len(ids), ids.ctypes.data,
                                         C.byref(bt), _ptr(out[:1]), _ptr(out[1:]), 1, stream_ptr())

    bad_row = row.copy()
    bad_row[rep.packer.offsets[2]:rep.packer.offsets[2] + 4] = np.frombuffer(np.int32(A).tobytes(), np.uint8)
    assert lib.xtb_episode_replay_add(rep.handle, 0, row.ctypes.data, row.nbytes - 16, stream_ptr()) == -1
    assert lib.xtb_episode_replay_add(rep.handle, BUF, row.ctypes.data, row.nbytes, stream_ptr()) == -1
    assert lib.xtb_episode_replay_add(rep.handle, 0, bad_row.ctypes.data, bad_row.nbytes, stream_ptr()) == -1
    assert gather([0, 1, B]) == -1                       # an id past the stored count
    assert gather([0, -1, 1]) == -1
    assert gather([0, 1], n=0) == -1
    assert gather(list(range(B)) + [0]) == -1            # more ids than stored episodes
    assert train([0, 1, 2]) == -1                        # not the model's batch
    assert train([0, 1, 2, B + 1]) == -1
    other = DeviceEpisodeReplay(alg.scheme, alg.groups, BUF, L + 1, alg.preprocess, True, False)   # inputs of another width
    for d in stream:
        other.insert_episode_batch(EpisodeBatch(alg.scheme, alg.groups, 1, L + 1, data=dict(d)))
    assert train(list(range(B)), replay=other) == -1
    assert lib.xtb_launch_count() == launches
    with one_rank_comm():
        assert lib.xtb_episode_replay_add(rep.handle, 0, row.ctypes.data, row.nbytes, stream_ptr()) == -3
        assert gather(list(range(B))) == -3
        assert train(list(range(B))) == -3
        with pytest.raises(RuntimeError, match="error -3"):
            algs["scc"].train(episode_num=9)
        with pytest.raises(RuntimeError, match="error -3"):
            alg.prepare_data(stream[0])
        assert (rep.buffer_index, rep.episodes_in_buffer) == (B, B)   # the refused store left the ring as it was
    assert lib.xtb_launch_count() == launches
    assert gather(list(range(B))) == 0 and train(list(range(B))) == 0
