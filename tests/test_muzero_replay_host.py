"""The Muzero learner's device replay, host side (no GPU): DEVICE_REPLAY / DEVICE_REPLAY_STEPS are checked before anything
touches CUDA; PoolPlanner against a step-by-step simulation of the pool; the host restatement of the device rules
(muzero_replay_oracle.py) against the reference learner's golden session, and its eviction rules."""
import os
import random

import numpy as np
import pytest
import torch

from muzero_replay_oracle import RestatedReplay
from xingtian_b200.algorithm import muzero as mz

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "muzero.npz"))
FIELDS = ("cur_state", "action", "reward", "child_visits", "target_value")
INFO = {"actor": {"model_name": "MuzeroMlp", "state_dim": [4], "action_dim": 3, "model_config": {"max_batch": 8}}}


class _Reached(Exception):
    pass


@pytest.mark.parametrize("cfg", [{"DEVICE_REPLAY": 1}, {"DEVICE_REPLAY": "yes"}, {"DEVICE_REPLAY": None},
                                 {"DEVICE_REPLAY": True, "DEVICE_REPLAY_STEPS": 0},
                                 {"DEVICE_REPLAY": True, "DEVICE_REPLAY_STEPS": -3},
                                 {"DEVICE_REPLAY": True, "DEVICE_REPLAY_STEPS": 2.5},
                                 {"DEVICE_REPLAY": True, "DEVICE_REPLAY_STEPS": True},
                                 {"DEVICE_REPLAY": False, "DEVICE_REPLAY_STEPS": "100"}])
def test_config_is_checked_before_cuda(cfg, monkeypatch):
    def touched(*a, **k):
        raise _Reached()
    monkeypatch.setattr(mz.Algorithm, "__init__", touched)
    cuda_before = torch.cuda.is_initialized()
    with pytest.raises(ValueError):
        mz.Muzero(INFO, dict(cfg, instance_num=1))
    assert torch.cuda.is_initialized() == cuda_before
    # a valid configuration gets past the checks to the model construction
    with pytest.raises(_Reached):
        mz.Muzero(INFO, {"DEVICE_REPLAY": True, "DEVICE_REPLAY_STEPS": 100})
    with pytest.raises(_Reached):
        mz.Muzero(INFO, {"DEVICE_REPLAY": np.bool_(False)})


def _simulate(size, steps, lengths):
    """PoolPlanner step by step against an explicit pool: every placement lies inside the pool and overwrites only
    the steps of the trajectories it evicts; evicted trajectories are the oldest stored ones; a live trajectory's steps
    are untouched from its placement until it leaves."""
    pl = mz.PoolPlanner(size, steps)
    owner = np.full(steps, -1)          # insertion number of the trajectory whose steps each pool step holds
    stored = {}                         # slot -> insertion number, live or evicted
    live = []                           # insertion numbers of live trajectories, oldest first
    for n, L in enumerate(lengths):
        slot, off, e0, ne = pl.place(L)
        assert slot == n % size and 0 <= off and off + L <= steps
        gone = [stored[slot]] if slot in stored and stored[slot] in live else []
        evicted = [stored[(e0 + k) % size] for k in range(ne)]
        assert slot not in [(e0 + k) % size for k in range(ne)]
        live = [x for x in live if x not in gone]
        assert live[:ne] == evicted, (n, live, evicted)        # the oldest live trajectories go first
        live = live[ne:]
        assert not set(owner[off:off + L]) & set(live)         # nothing live is overwritten
        owner[off:off + L] = n
        stored[slot] = n
        live.append(n)
        assert [pl.fifo[i] for i in range(len(pl.fifo))] == [x % size for x in live]
        for x in live:                                          # every live trajectory still owns its steps
            s = x % size
            assert pl.live[s] and (owner[pl.off[s]:pl.off[s] + pl.len[s]] == x).all()
    return pl


@pytest.mark.parametrize("size,steps,seed", [(8, 64, 0), (16, 300, 1), (50, 1000, 2), (5, 40, 3), (30, 30, 4)])
def test_planner_against_pool_simulation(size, steps, seed):
    rng = np.random.default_rng(seed)
    lengths = [int(x) for x in rng.integers(1, min(steps, 60) + 1, 400)]
    pl = _simulate(size, steps, lengths)
    assert pl.evictions > 0 and pl.count == size


def test_planner_without_pressure_never_evicts():
    rng = np.random.default_rng(7)
    pl = _simulate(12, 100000, [int(x) for x in rng.integers(7, 300, 200)])
    assert pl.evictions == 0
    with pytest.raises(ValueError):
        pl.place(100001)


def test_restatement_is_the_reference_learner_without_evictions():
    ref = RestatedReplay(8, 4096, 5)
    trajs = [{k: GOLD["traj%d_%s" % (t, k)] for k in FIELDS} for t in range(22)]
    random.seed(1234)
    step = 0
    for t, tr in enumerate(trajs):
        if len(tr["reward"]) > 6:
            ref.add(dict(tr, traj_id=t), 0.01 * tr["cur_state"].sum(1))
        if t in (3, 12, 21):
            for _ in range(3):
                if len(ref) < 6:
                    continue
                slots, pos = ref.draw([random.random() for _ in range(12)])
                img, act, tv, tr_, tp = ref.gather(slots, pos)
                for name, got in (("image", img), ("action", act), ("tv", tv), ("tr", tr_), ("tp", tp)):
                    np.testing.assert_array_equal(got, GOLD["step%d_%s" % (step, name)])
                ref.update(slots, pos, 0.01 * img.sum(1))
                step += 1
    assert step == int(GOLD["n_train_steps"]) and ref.planner.evictions == 0
    assert [d["traj_id"] for d in ref.buff.storage] == list(GOLD["buf_ids"])
    np.testing.assert_array_equal(ref.traj_leaves(), GOLD["buf_pri"])
    np.testing.assert_array_equal(np.concatenate([ref.pos_leaves(s) for s in range(len(ref))]), GOLD["buf_pos_pri"])


def test_evicted_slots_are_never_revived_or_drawn():
    ref = RestatedReplay(16, 200, 5)
    rng = np.random.default_rng(5)
    random.seed(3)
    for t in range(120):
        L = int(rng.integers(7, 50))
        obs = rng.normal(size=(L, 4))
        ref.add(dict(cur_state=obs, action=rng.integers(0, 3, L), reward=rng.normal(size=L), child_visits=rng.dirichlet(np.ones(3), L),
                     target_value=rng.normal(size=L)), 0.01 * obs.sum(1))
        if len(ref) >= 16:
            slots, pos = ref.draw([random.random() for _ in range(32)])
            assert all(ref.planner.live[s] for s in slots)
            ref.update(slots, pos, 0.01 * ref.gather(slots, pos)[0].sum(1))
            dead = [s for s in range(16) if not ref.planner.live[s]]
            assert all(ref.buff.it_sum[s] == 0.0 for s in dead)
    assert ref.planner.evictions > 20


def test_plan_changes_nothing_until_commit():
    """DeviceTrajectoryReplay asks plan() first and commits only once the device stored the trajectory, so a failed store
    leaves the planner where it was."""
    pl = mz.PoolPlanner(6, 120)
    rng = np.random.default_rng(9)

    def snapshot():
        return (pl.next_idx, pl.count, pl.head, pl.evictions, list(pl.off), list(pl.len), list(pl.live), list(pl.fifo))
    for _ in range(200):
        L = int(rng.integers(7, 50))
        before = snapshot()
        placement = pl.plan(L)
        assert snapshot() == before and pl.plan(L) == placement
        pl.commit(placement, L)
    assert pl.evictions > 0
