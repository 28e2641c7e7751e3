"""The Muzero learner's replay on the H100 (DeviceTrajectoryReplay, xtb_muzero_replay_*): the device primitives replay the
muzero.npz session (the reference learner's own draws, minibatches and priorities) bit for bit; the device learner
against the host learner on the real models; eviction against the host restatement (muzero_replay_oracle.py); graph
replay against eager launches; argument checks that launch nothing."""
import ctypes as C
import os
import random
import warnings

import numpy as np
import pytest
import torch

from muzero_replay_oracle import RestatedReplay
from test_gpu_kernels import one_rank_comm

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "muzero.npz"))
FIELDS = ("cur_state", "action", "reward", "child_visits", "target_value")


def _stand_in(obs):
    """the fixture's stand-in model: value = 0.01 * sum of the observation row"""
    return 0.01 * np.asarray(obs, np.float64).reshape(len(obs), -1).sum(1)


def _replay(size, steps, B, K=5, A=3, obs_shape=(4,)):
    from xingtian_b200.algorithm.muzero import DeviceTrajectoryReplay
    torch.cuda.set_device(0)
    return DeviceTrajectoryReplay(size, steps, obs_shape, np.float32, A, K, B, torch.device("cuda", 0))


def _check_trees(dev, ref):
    st = dev.state()
    n = len(ref)
    assert st["count"] == n
    np.testing.assert_array_equal(st["traj_tree"][st["leaves"]:st["leaves"] + n], ref.traj_leaves())
    for s in range(n):
        if ref.planner.live[s]:
            np.testing.assert_array_equal(dev.position_leaves(st, s), ref.pos_leaves(s))
    return st


def test_primitives_replay_the_golden_session():
    dev = _replay(8, 4096, 6)
    ref = RestatedReplay(8, 4096, 5)
    trajs = [{k: GOLD["traj%d_%s" % (t, k)] for k in FIELDS} for t in range(22)]
    ids = [None] * 8
    random.seed(1234)
    step = 0
    for t, tr in enumerate(trajs):
        if len(tr["reward"]) > 6:
            v = _stand_in(tr["cur_state"])
            ids[dev.add(tr, values=v)] = t
            ref.add(tr, v)
        if t in (3, 12, 21):
            for _ in range(3):
                if len(dev) < 6:
                    continue
                u = [random.random() for _ in range(12)]
                slot, pos, obs, action, tv, tr_, tp = (x.cpu().numpy() for x in dev.sample(u))
                assert (list(slot), list(pos)) == ref.draw(u)
                np.testing.assert_array_equal(obs, GOLD["step%d_image" % step].astype(np.float32))
                np.testing.assert_array_equal(action, GOLD["step%d_action" % step])
                np.testing.assert_array_equal(tv, GOLD["step%d_tv" % step].astype(np.float32))
                np.testing.assert_array_equal(tr_, GOLD["step%d_tr" % step].astype(np.float32))
                np.testing.assert_array_equal(tp, GOLD["step%d_tp" % step].astype(np.float32))
                values = _stand_in(GOLD["step%d_image" % step])
                assert dev.update(torch.from_numpy(slot).cuda(), torch.from_numpy(pos).cuda(), values) == 0
                ref.update(list(slot), list(pos), values)
                step += 1
    assert step == int(GOLD["n_train_steps"])
    st = _check_trees(dev, ref)
    assert len(dev) == int(GOLD["buf_len"]) and [ids[s] for s in range(len(dev))] == list(GOLD["buf_ids"])
    L = st["leaves"]
    np.testing.assert_array_equal(st["traj_tree"][L:L + len(dev)], GOLD["buf_pri"])
    np.testing.assert_array_equal(np.concatenate([dev.position_leaves(st, s) for s in range(len(dev))]), GOLD["buf_pos_pri"])


def _traj(rng, L, A, obs_shape, kind):
    if kind == "float32":
        obs = rng.normal(size=(L,) + obs_shape).astype(np.float32)
    else:
        obs = rng.integers(0, 256, (L,) + obs_shape).astype(np.uint8)
    return dict(cur_state=obs, action=rng.integers(0, A, L), reward=rng.uniform(0, 3, L).round(2), done=np.zeros(L, bool),
                child_visits=rng.dirichlet(np.ones(A), L), target_value=rng.uniform(0, 8, L))


def _learners(name, obs_shape, A, obs_type, B, size, max_batch, graph=True, steps=1 << 15):
    from xingtian_b200 import alg_builder
    torch.cuda.set_device(0)
    mc = {"max_batch": max_batch, "init_seed": 3, "value_min": 0, "value_max": 10, "reward_min": 0, "reward_max": 4,
          "obs_type": obs_type, "use_cuda_graph": graph}
    info = {"actor": {"model_name": name, "state_dim": list(obs_shape), "action_dim": A, "model_config": mc}}
    cfg = {"instance_num": 1, "agent_num": 1, "BATCH_SIZE": B, "BUFFER_SIZE": size, "UNROLL_STEP": 5}
    host = alg_builder("Muzero", info, cfg)
    dev = alg_builder("Muzero", info, dict(cfg, DEVICE_REPLAY=True, DEVICE_REPLAY_STEPS=steps))
    return host, dev


def _host_draw(host, seed):
    random.seed(seed)
    state = random.getstate()
    trajs, pos, *_ = host.sample_batch()
    random.setstate(state)
    ids = [id(t) for t in host.buff.storage]
    return [ids.index(id(t)) for t in trajs], list(pos)


def _compare(host, dev, trajs, n_steps, exact=True):
    """Both learners over the same trajectories and host draws: identical (slot, position) draws and losses at every step;
    parameters and trees bitwise when `exact`, else to float32 rounding (see the B = 64 case)."""
    for tr in trajs:
        host.prepare_data(dict(tr))
        dev.prepare_data(dict(tr))
    ref = host.buff
    assert len(ref) >= host.batch_size
    same = np.testing.assert_array_equal if exact else lambda a, b: np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)
    st = dev.buff.state()
    assert st["count"] == len(ref)
    np.testing.assert_array_equal(st["traj_tree"][st["leaves"]:st["leaves"] + len(ref)], [ref.it_sum[i] for i in range(len(ref))])
    draws = []
    for s in range(n_steps):
        slots, pos = _host_draw(host, 50 + s)
        loss_h = host.train()
        random.seed(50 + s)
        loss_d = dev.train()
        b = dev.buff.buffers(dev.batch_size)
        assert (list(b["slot"].cpu().numpy()), list(b["pos"].cpu().numpy())) == (slots, pos), s
        assert loss_h == loss_d, (s, loss_h, loss_d)
        same(dev.actor.params.cpu().numpy(), host.actor.params.cpu().numpy())
        draws.append((slots, pos))
    st = dev.buff.state()
    L = st["leaves"]
    same(st["traj_tree"][L:L + len(ref)], [ref.it_sum[i] for i in range(len(ref))])
    for s in range(len(ref)):
        pb = ref.storage[s]["pos_buff"]
        same(dev.buff.position_leaves(st, s), [pb.it_sum[i] for i in range(len(pb))])
    return draws


@pytest.mark.parametrize("B", [1, 8, 64])
def test_mlp_device_learner_matches_host_learner(B):
    """B = 64 fills max_batch.  There the fp32 weight gradient of the first dense layers splits the batch with atomics, so
    two runs of the same step (host replay or device replay alike) agree to rounding only: the first step's draws and loss
    are compared bitwise, then parameters and trees to rounding.  test_mlp_full_batch_bitwise_over_steps checks the
    replay at this batch bit for bit over several steps."""
    host, dev = _learners("MuzeroMlp", (4,), 3, "float32", B, 96, 64)
    rng = np.random.default_rng(B)
    lengths = [7, 2100, 9] + [int(x) for x in rng.integers(7, 60, 90)]
    _compare(host, dev, [_traj(rng, L, 3, (4,), "float32") for L in lengths], 4 if B <= 8 else 1, exact=B <= 8)


def test_mlp_full_batch_bitwise_over_steps():
    """B = max_batch = 64 over several steps, bit for bit: the device learner's draws and both tree levels after every
    step against the host restatement fed with the device learner's own post-step values (value inference of the
    gathered batch with the updated weights, the launches the step's value output runs).  One heavy trajectory makes
    trajectories and (trajectory, position) pairs repeat within a step.  This checks the replay at a full batch without
    the rounding the weight gradient's atomics leave between two runs of the model step."""
    _, dev = _learners("MuzeroMlp", (4,), 3, "float32", 64, 96, 64)
    ref = RestatedReplay(96, 1 << 15, 5)
    rng = np.random.default_rng(11)
    lengths = [7, 2100, 9] + [int(x) for x in rng.integers(7, 60, 90)]
    trajs = [_traj(rng, L, 3, (4,), "float32") for L in lengths]
    trajs[0]["target_value"] = trajs[0]["target_value"] + 400.0
    for tr in trajs:
        dev.prepare_data(dict(tr))
        ref.add(tr, dev.actor.value_inference(tr["cur_state"]))
    _check_trees(dev.buff, ref)
    repeats = []
    for step in range(4):
        random.seed(70 + step)
        u = [random.random() for _ in range(128)]
        random.seed(70 + step)
        dev.train()
        b = dev.buff.buffers(64)
        slots, pos = ref.draw(u)
        assert (list(b["slot"].cpu().numpy()), list(b["pos"].cpu().numpy())) == (slots, pos), step
        ref.update(slots, pos, dev.actor.value_inference(b["obs"].cpu().numpy()))
        _check_trees(dev.buff, ref)
        repeats.append(len(set(zip(slots, pos))) < len(slots))
    assert all(repeats)


def test_mlp_repeated_trajectories_and_pairs():
    """eight trajectories of two positions each, one of them with a far larger weight, for a batch of 8: trajectories and
    (trajectory, position) pairs repeat within a step, so the order of its updates matters"""
    host, dev = _learners("MuzeroMlp", (4,), 3, "float32", 8, 8, 8)
    rng = np.random.default_rng(1)
    trajs = [_traj(rng, 7, 3, (4,), "float32") for _ in range(8)]
    trajs[2]["target_value"] = trajs[2]["target_value"] + 50.0
    draws = _compare(host, dev, trajs, 4)
    slots, pos = draws[0]
    assert len(set(slots)) < len(slots) and len(set(zip(slots, pos))) < len(slots)


@pytest.mark.parametrize("obs_type", ["uint8", "int8"])
def test_cnn_device_learner_matches_host_learner(obs_type):
    host, dev = _learners("MuzeroCnn", (84, 84, 4), 4, obs_type, 8, 12, 8)
    rng = np.random.default_rng(7)
    _compare(host, dev, [_traj(rng, L, 4, (84, 84, 4), "uint8") for L in (7, 40, 9, 2100, 30, 12, 8, 7, 25, 11)], 3)


def test_eviction_against_the_restatement():
    """A pool that forces evictions: the device primitives against the host restatement with the stand-in values, bit for
    bit through many evictions; no evicted slot is drawn and its leaf stays 0."""
    dev = _replay(16, 300, 12)
    ref = RestatedReplay(16, 300, 5)
    rng = np.random.default_rng(4)
    random.seed(9)
    for t in range(70):
        L = int(rng.integers(7, 90))
        tr = _traj(rng, L, 3, (4,), "float32")
        v = _stand_in(tr["cur_state"])
        assert dev.add(tr, values=v) == ref.add(tr, v)
        if len(dev) >= 12 and t % 3 == 0:
            u = [random.random() for _ in range(24)]
            slot, pos = (x.cpu().numpy() for x in dev.sample(u)[:2])
            rs, rp = ref.draw(u)
            assert (list(slot), list(pos)) == (rs, rp)
            assert all(ref.planner.live[s] for s in rs)
            img = ref.gather(rs, rp)[0]
            dev.update(torch.from_numpy(slot).cuda(), torch.from_numpy(pos).cuda(), _stand_in(img))
            ref.update(rs, rp, _stand_in(img))
    assert ref.planner.evictions > 10
    st = _check_trees(dev, ref)
    dead = [s for s in range(len(ref)) if not ref.planner.live[s]]
    assert dead and all(st["traj_tree"][st["leaves"] + s] == 0.0 for s in dead)
    np.testing.assert_array_equal(st["live"][:len(ref)], ref.planner.live[:len(ref)])


def test_learner_evicts_warns_once_and_never_draws_evicted():
    host, dev = _learners("MuzeroMlp", (4,), 3, "float32", 8, 20, 8, steps=200)
    rng = np.random.default_rng(2)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        for t in range(60):
            dev.prepare_data(_traj(rng, int(rng.integers(7, 40)), 3, (4,), "float32"))
            if t >= 10:
                dev.train()
                live = dev.buff.planner.live
                slots = dev.buff.buffers(8)["slot"].cpu().numpy()
                assert all(live[s] for s in slots)
    assert sum(issubclass(x.category, RuntimeWarning) for x in w) == 1
    st = dev.buff.state()
    dead = [s for s in range(len(dev.buff)) if not dev.buff.planner.live[s]]
    assert dead and all(st["traj_tree"][st["leaves"] + s] == 0.0 for s in dead)
    with pytest.raises(ValueError):
        dev.prepare_data(_traj(rng, 201, 3, (4,), "float32"))


def test_graph_replay_matches_eager_and_captures_once():
    from xingtian_b200 import capi
    lib = capi.lib()
    _, g = _learners("MuzeroMlp", (4,), 3, "float32", 8, 24, 8, graph=True, steps=400)
    _, e = _learners("MuzeroMlp", (4,), 3, "float32", 8, 24, 8, graph=False, steps=400)
    rng = np.random.default_rng(6)
    trajs = [_traj(rng, int(rng.integers(7, 40)), 3, (4,), "float32") for _ in range(80)]
    c0 = None
    for t, tr in enumerate(trajs):
        for alg in (g, e):
            alg.prepare_data(dict(tr))
        if t >= 8:
            losses = []
            for alg in (g, e):
                random.seed(t)
                losses.append(alg.train())
            assert (g.buff.buffers(8)["slot"].cpu().numpy() == e.buff.buffers(8)["slot"].cpu().numpy()).all()
            assert abs(losses[0] - losses[1]) <= 1e-5 * max(1.0, abs(losses[1]))
            if c0 is None:
                c0 = lib.xtb_graph_capture_count()
    assert g.buff.planner.evictions > 0 and len(g.buff) == 24        # the ring wrapped and the pool evicted
    assert lib.xtb_graph_capture_count() == c0


def test_invalid_arguments_launch_nothing():
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    lib = capi.lib()
    _, alg = _learners("MuzeroMlp", (4,), 3, "float32", 4, 8, 8, steps=100)
    r, m = alg.buff, alg.actor
    b = r.buffers(4)
    scratch = torch.zeros(4096, dtype=torch.float64, device="cuda")
    p = _ptr(scratch)
    torch.cuda.synchronize()
    n0 = lib.xtb_launch_count()
    out = C.c_void_p()
    assert lib.xtb_muzero_replay_create(0, 100, 5, 16, 3, 8, C.byref(out)) == -1
    assert lib.xtb_muzero_replay_create(8, 100, 5, 16, 1025, 8, C.byref(out)) == -1
    assert lib.xtb_muzero_replay_create(8, 0, 5, 16, 3, 8, C.byref(out)) == -1

    def add(slot=0, off=0, e0=0, ne=0, L=10, values=p, model=None):
        return lib.xtb_muzero_replay_add(r.handle, model, slot, off, e0, ne, p, p, p, p, p, L, values, stream_ptr())
    assert add(L=6) == -1                    # not longer than K + 1
    assert add(L=101) == -1                  # longer than the pool
    assert add(off=95) == -1                 # past the pool's end
    assert add(slot=8) == -1
    assert add(slot=2, e0=1, ne=2) == -1     # evicts its own slot
    assert add(values=None) == -1            # neither values nor a model
    train = lambda B: lib.xtb_muzero_replay_train(r.handle, m.handle, m.opt.handle, B, _ptr(b["u"]), _ptr(b["slot"]), _ptr(b["pos"]),
                                                  C.byref(b["batch"]), 0.0, _ptr(b["loss"]), _ptr(b["status"]), 1, stream_ptr())
    assert train(4) == -3                    # nothing stored yet
    assert lib.xtb_muzero_replay_sample(r.handle, 0, _ptr(b["u"]), _ptr(b["slot"]), _ptr(b["pos"]), C.byref(b["batch"]), stream_ptr()) == -1
    assert lib.xtb_muzero_replay_update(r.handle, 9, _ptr(b["slot"]), _ptr(b["pos"]), p, stream_ptr()) == -1
    with one_rank_comm():
        assert add() == -3 and b"data-parallel" in lib.xtb_last_error()
        assert lib.xtb_muzero_replay_update(r.handle, 4, _ptr(b["slot"]), _ptr(b["pos"]), p, stream_ptr()) == -3
    with pytest.raises(ValueError):
        alg.prepare_data(_traj(np.random.default_rng(0), 101, 3, (4,), "float32"))
    torch.cuda.synchronize()
    assert lib.xtb_launch_count() == n0
    # a failed add leaves the planner where it was
    planner = (r.planner.next_idx, r.planner.count, r.planner.head, list(r.planner.fifo))
    with one_rank_comm():
        with pytest.raises(RuntimeError):
            alg.prepare_data(_traj(np.random.default_rng(0), 10, 3, (4,), "float32"))
    assert (r.planner.next_idx, r.planner.count, r.planner.head, list(r.planner.fifo)) == planner and len(r) == 0
    torch.cuda.synchronize()
    assert lib.xtb_launch_count() == n0
    # updates write the trajectory leaf of every batch position: a batch past the stored slots is refused, as the host's
    # update_priorities refuses it, here with max_batch 8 above the ring's 8 slots not yet filled
    rng = np.random.default_rng(1)
    for _ in range(2):
        alg.prepare_data(_traj(rng, 10, 3, (4,), "float32"))
    torch.cuda.synchronize()
    n1 = lib.xtb_launch_count()
    assert lib.xtb_muzero_replay_update(r.handle, 3, _ptr(b["slot"]), _ptr(b["pos"]), p, stream_ptr()) == -1
    assert b"stored slots" in lib.xtb_last_error()
    assert train(3) == -1 and b"stored slots" in lib.xtb_last_error()
    # a replay with fewer slots than max_batch
    small = _replay(2, 100, 8)
    for _ in range(2):
        tr = _traj(rng, 10, 3, (4,), "float32")
        small.add(tr, values=_stand_in(tr["cur_state"]))
    torch.cuda.synchronize()
    n2 = lib.xtb_launch_count()
    assert lib.xtb_muzero_replay_update(small.handle, 3, _ptr(b["slot"]), _ptr(b["pos"]), p, stream_ptr()) == -1
    assert lib.xtb_launch_count() == n2
    # a trainer whose model reads other observations than the replay stores
    _, other = _learners("MuzeroMlp", (6,), 3, "float32", 4, 8, 8, steps=100)
    for _ in range(2):
        alg.prepare_data(_traj(rng, 10, 3, (4,), "float32"))
    torch.cuda.synchronize()
    n3 = lib.xtb_launch_count()
    assert lib.xtb_muzero_replay_train(r.handle, other.actor.handle, other.actor.opt.handle, 4, _ptr(b["u"]), _ptr(b["slot"]),
                                       _ptr(b["pos"]), C.byref(b["batch"]), 0.0, _ptr(b["loss"]), _ptr(b["status"]), 1,
                                       stream_ptr()) == -1
    assert b"does not match" in lib.xtb_last_error()
    assert lib.xtb_launch_count() == n3
    assert n1 >= n0 and len(r) == 4


def test_nan_priority_stops_the_updates():
    """A NaN post-step value: the entries before it are applied, it and every later entry are not."""
    from xingtian_b200 import capi
    dev = _replay(8, 400, 4)
    rng = np.random.default_rng(3)
    trajs = [_traj(rng, 12, 3, (4,), "float32") for _ in range(5)]
    for tr in trajs:                                # slots 0 .. 4 in order
        dev.add(tr, values=_stand_in(tr["cur_state"]))
    slot, pos = dev.sample([0.3, 0.6, 0.1, 0.9, 0.5, 0.5, 0.5, 0.5])[:2]
    s, p = [int(x) for x in slot.cpu()], [int(x) for x in pos.cpu()]
    before = dev.state()
    status = dev.update(slot, pos, [1e6, float("nan"), 2e6, 3e6])
    assert status & capi.MZR_BAD_PRIORITY and status == dev.status()
    after = dev.state()
    L = after["leaves"]
    changed = np.nonzero(after["traj_tree"][L:L + 8] != before["traj_tree"][L:L + 8])[0]
    assert list(changed) == [0]                     # entry 0's batch-position leaf, and no other
    for j in range(5):                              # position leaves: only entry 0's leaf moved
        moved = list(np.nonzero(dev.position_leaves(after, j) != dev.position_leaves(before, j))[0])
        assert moved == ([p[0]] if j == s[0] else []), (j, moved)
    assert dev.position_leaves(after, s[0])[p[0]] == abs(1e6 - float(trajs[s[0]]["target_value"][p[0]]))
    # batch-position leaf 0 took slot s[0]'s weight after that write: its tree root over its 7 positions
    assert after["traj_tree"][L] == after["forest"][4 * int(after["off"][s[0]]) + 1] / 7


def test_learner_raises_value_error_on_nan_priority():
    """The learner turns the device's XTB_MZR_BAD_PRIORITY into the host's ValueError.  The model's value head clips its
    output into the value range (NaN included), so the step is followed here by a real device update from NaN values,
    whose status the learner then reads; that update applies nothing."""
    _, dev = _learners("MuzeroMlp", (4,), 3, "float32", 4, 8, 8, steps=400)
    rng = np.random.default_rng(8)
    for _ in range(6):
        dev.prepare_data(_traj(rng, 12, 3, (4,), "float32"))
    step, snap = dev.buff.train, {}

    def step_then_nan_update(model, uniforms):
        loss, status = step(model, uniforms)
        assert status == 0
        b = dev.buff.buffers(4)
        snap["before"] = dev.buff.state()
        return loss, dev.buff.update(b["slot"], b["pos"], [float("nan")] * 4)
    dev.buff.train = step_then_nan_update
    random.seed(0)
    with pytest.raises(ValueError, match="not > 0"):
        dev.train()
    after = dev.buff.state()
    np.testing.assert_array_equal(after["traj_tree"], snap["before"]["traj_tree"])
    np.testing.assert_array_equal(after["forest"], snap["before"]["forest"])
