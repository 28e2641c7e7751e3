"""The Muzero learner (xt/algorithm/muzero/muzero.py) over MuzeroCnn / MuzeroMlp.

Trajectories live on the host in a proportional prioritised buffer (segment trees written for this package with the query
semantics the reference's learner relies on); each training call samples BATCH_SIZE trajectories and one position per
trajectory, gathers the observation, the UNROLL_STEP actions and the UNROLL_STEP + 1 targets of every sample, uploads the
minibatch through the staged pinned copy and runs one model step, which also returns the post-update values used as
the new priorities.  With alg_config DEVICE_REPLAY the same rules run on the device (DeviceTrajectoryReplay)."""
import ctypes as C
import numbers
import operator
import random
import warnings
from collections import deque
from itertools import islice

import numpy as np
import torch

from .. import capi
from ..capi import check, lib
from ..engine import _ptr, stage_h2d, stream_ptr
from ..registry import Registers, import_config
from .base import Algorithm

# xt/algorithm/muzero/default_config.py
BATCH_SIZE = 1024
BUFFER_SIZE = 100000
GAMMA = 0.997
TD_STEP = 10
UNROLL_STEP = 5
# pool steps of the device replay when alg_config sets DEVICE_REPLAY but not DEVICE_REPLAY_STEPS (both keys are read from
# each learner's alg_config, not through import_config, so one learner's choice does not leak into the next)
_DEFAULT_REPLAY_STEPS = 1 << 16


class SegmentTree(object):
    """Array segment tree over `capacity` (a power of two) leaves; node i holds op(node 2i, node 2i+1).

    reduce(start, end) combines leaves start .. end - 1 (end None: the whole tree; negative: from the back), splitting the
    range at the node midpoints, so sums are formed in the same order for the same range."""

    def __init__(self, capacity, op, neutral):
        if capacity <= 0 or capacity & (capacity - 1):
            raise ValueError("capacity must be a positive power of 2")
        self.capacity, self.op = capacity, op
        self.value = [neutral] * (2 * capacity)

    def __setitem__(self, i, v):
        i += self.capacity
        self.value[i] = v
        i //= 2
        while i >= 1:
            self.value[i] = self.op(self.value[2 * i], self.value[2 * i + 1])
            i //= 2

    def __getitem__(self, i):
        return self.value[self.capacity + i]

    def _reduce(self, lo, hi, node, nlo, nhi):
        if lo == nlo and hi == nhi:
            return self.value[node]
        mid = (nlo + nhi) // 2
        if hi <= mid:
            return self._reduce(lo, hi, 2 * node, nlo, mid)
        if lo > mid:
            return self._reduce(lo, hi, 2 * node + 1, mid + 1, nhi)
        return self.op(self._reduce(lo, mid, 2 * node, nlo, mid), self._reduce(mid + 1, hi, 2 * node + 1, mid + 1, nhi))

    def reduce(self, start=0, end=None):
        end = self.capacity if end is None else (end + self.capacity if end < 0 else end)
        return self._reduce(start, end - 1, 1, 0, self.capacity - 1)


class SumTree(SegmentTree):
    def __init__(self, capacity):
        super().__init__(capacity, operator.add, 0.0)

    def find_prefixsum_idx(self, mass):
        """the leaf where the running sum first exceeds `mass`"""
        i = 1
        while i < self.capacity:
            if self.value[2 * i] > mass:
                i = 2 * i
            else:
                mass -= self.value[2 * i]
                i = 2 * i + 1
        return i - self.capacity


class PrioritizedBuffer(object):
    """Proportional prioritised ring of `size` items (xt/algorithm/prioritized_replay_buffer_muzero.py semantics).

    sample() draws one random.random() per item, in order, and takes the total of leaves 0 .. len - 2 as the mass to
    spread (the reference's sum(0, len - 1) with its exclusive end): the newest slot of a full range is never drawn unless
    the masses overshoot into it.  weight() is the mean priority over the stored items."""

    def __init__(self, size, alpha=1.0):
        cap = 1
        while cap < size:
            cap *= 2
        self.size, self.alpha = size, alpha
        self.storage, self.next_idx = [], 0
        self.it_sum, self.it_min, self.it_max = SumTree(cap), SegmentTree(cap, min, float("inf")), SegmentTree(cap, max, 0.0)
        self.max_priority = 1.0

    def __len__(self):
        return len(self.storage)

    def _set(self, i, priority):
        p = priority ** self.alpha
        self.it_sum[i] = p
        self.it_min[i] = p
        self.it_max[i] = p

    def add(self, data, priority=None):
        i = self.next_idx
        if i >= len(self.storage):
            self.storage.append(data)
        else:
            self.storage[i] = data
        self.next_idx = (i + 1) % self.size
        self._set(i, self.max_priority if priority is None else priority)
        return i

    def sample(self, batch_size, beta):
        total = self.it_sum.reduce(0, len(self.storage) - 1)
        step = total / batch_size
        idxes = [self.it_sum.find_prefixsum_idx(random.random() * step + k * step) for k in range(batch_size)]
        whole, n = self.it_sum.reduce(), len(self.storage)
        p_min = max(self.it_min.reduce() / whole, 1e-5)
        max_w = (p_min * n) ** (-beta)
        weights = np.array([((self.it_sum[i] / whole) * n) ** (-beta) / max_w for i in idxes])
        return [self.storage[i] for i in idxes], weights, idxes

    def update_priorities(self, idxes, priorities):
        for i, p in zip(idxes, priorities):
            if not (p > 0 and 0 <= i < len(self.storage)):
                raise ValueError("priority update {} at {} out of range".format(p, i))
            self._set(i, p)
            self.max_priority = max(self.max_priority, p)

    def weight(self):
        return self.it_sum.reduce() / len(self.storage) if self.storage else 0


class PoolPlanner(object):
    """Where DeviceTrajectoryReplay puts each trajectory: slot next_idx of a `size`-slot ring, as PrioritizedBuffer.add,
    and a contiguous range of a `steps`-step pool, taken in insertion order from `head` (from 0 when the rest of the pool
    is too short).  Trajectories still stored in the way are evicted, oldest first: those past `head` when the range
    starts over at 0, then those overlapping the range.  They are the oldest stored ones, the slots the ring would
    overwrite next.  plan() -> (slot, offset, first evicted slot, evicted count), the evicted slots consecutive in the
    ring; commit() records it once the trajectory is stored; place() does both."""

    def __init__(self, size, steps):
        self.size, self.steps = int(size), int(steps)
        self.next_idx = self.count = self.head = self.evictions = 0
        self.off, self.len, self.live = [0] * self.size, [0] * self.size, [False] * self.size
        self.fifo = deque()     # live slots, oldest first

    def plan(self, length):
        """Where a trajectory of `length` steps would go, without changing anything: (slot, offset, first evicted slot,
        evicted count)."""
        if not 0 < length <= self.steps:
            raise ValueError("a trajectory of {} steps does not fit a pool of {} (DEVICE_REPLAY_STEPS)".format(length, self.steps))
        s = self.next_idx
        # a live slot s is the oldest trajectory, which the ring overwrites: the candidates for eviction come after it
        queue = islice(self.fifo, 1 if self.live[s] else 0, None)
        wrap = self.head + length > self.steps
        off = 0 if wrap else self.head
        evicted = []
        for o in queue:
            lo, hi = self.off[o], self.off[o] + self.len[o]
            if not ((wrap and lo >= self.head) or (lo < off + length and off < hi)):
                break
            evicted.append(o)
        assert all(e == (evicted[0] + i) % self.size for i, e in enumerate(evicted))
        return s, off, (evicted[0] if evicted else 0), len(evicted)

    def commit(self, placement, length):
        """Record a placement plan(length) returned, once the trajectory is stored."""
        s, off, _, ne = placement
        assert s == self.next_idx
        if self.live[s]:
            assert self.fifo[0] == s
            self.fifo.popleft()
            self.live[s] = False
        for _ in range(ne):
            self.live[self.fifo.popleft()] = False
        self.off[s], self.len[s], self.live[s] = off, length, True
        self.fifo.append(s)
        self.head = off + length
        self.next_idx = (s + 1) % self.size
        self.count = max(self.count, s + 1)
        self.evictions += ne

    def place(self, length):
        placement = self.plan(length)
        self.commit(placement, length)
        return placement


class DeviceTrajectoryReplay(object):
    """The Muzero learner's replay in HBM (xtb_muzero_replay): a pool of `steps` steps for the trajectories of a
    `size`-slot ring, placed by PoolPlanner, with the host learner's two-level prioritized draw, gather and updates
    on the device.  Until the first eviction it holds exactly what PrioritizedBuffer would.  An evicted slot keeps
    its place in len(), its leaf is 0 and no draw or update revives it."""

    def __init__(self, size, steps, obs_shape, obs_dtype, n_actions, unroll, max_batch, device):
        self.obs_shape, self.obs_dtype = tuple(obs_shape), np.dtype(obs_dtype)
        self.A, self.K, self.max_batch, self.device = int(n_actions), int(unroll), int(max_batch), device
        self.row_bytes = int(np.prod(self.obs_shape)) * self.obs_dtype.itemsize
        self.planner = PoolPlanner(size, steps)
        self.handle = C.c_void_p()
        with torch.cuda.device(device):
            check(lib().xtb_muzero_replay_create(self.planner.size, self.planner.steps, self.K, self.row_bytes, self.A,
                                                 self.max_batch, C.byref(self.handle)))
        self._stage = None
        self._bufs = {}
        self._warned = False

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                lib().xtb_muzero_replay_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:   # interpreter shutdown
            pass

    def __len__(self):
        return self.planner.count

    def add(self, train_data, model=None, values=None):
        """Store one trajectory (cur_state, action, target_value, reward, child_visits of one length L > K + 1) with one
        staged upload.  Position priorities from `values` [L] when given, else from `model`'s value inference of the
        stored rows.  -> the slot.  ValueError, before any launch, when it is too short or longer than the pool."""
        L = len(train_data["reward"])
        if L <= self.K + 1:
            raise ValueError("a trajectory of {} steps is not longer than UNROLL_STEP + 1 = {}".format(L, self.K + 1))
        if L > self.planner.steps:
            raise ValueError("a trajectory of {} steps does not fit a pool of {} (DEVICE_REPLAY_STEPS)".format(L, self.planner.steps))
        obs = model._host_obs(train_data["cur_state"]) if model is not None else np.asarray(train_data["cur_state"], self.obs_dtype)
        parts = [np.ascontiguousarray(obs, self.obs_dtype).view(np.uint8).reshape(-1),
                 np.ascontiguousarray(train_data["action"], np.int32).reshape(-1).view(np.uint8),
                 np.ascontiguousarray(train_data["target_value"], np.float64).reshape(-1).view(np.uint8),
                 np.ascontiguousarray(train_data["reward"], np.float32).reshape(-1).view(np.uint8),
                 np.ascontiguousarray(train_data["child_visits"], np.float32).reshape(-1).view(np.uint8)]
        if values is not None:
            parts.append(np.ascontiguousarray(values, np.float64).reshape(-1).view(np.uint8))
        sizes = [L * self.row_bytes, L * 4, L * 8, L * 4, L * self.A * 4, L * 8][:len(parts)]
        if [p.size for p in parts] != sizes:
            raise ValueError("trajectory fields disagree with {} steps of {} bytes and {} actions".format(L, self.row_bytes, self.A))
        if values is None and model is None:
            raise ValueError("add() needs the model or the values")
        offs = np.cumsum([0] + [(n + 15) // 16 * 16 for n in sizes])
        host = np.zeros(int(offs[-1]), np.uint8)
        for o, p in zip(offs, parts):
            host[o:o + p.size] = p
        if self._stage is None or self._stage.numel() < host.size:
            self._stage = torch.empty(max(host.size, 1 << 20), dtype=torch.uint8, device=self.device)
        stage_h2d(self._stage[:host.size], host, np.uint8)
        placement = self.planner.plan(L)
        slot, off, e0, ne = placement
        p = [C.c_void_p(self._stage.data_ptr() + int(o)) for o in offs[:-1]]
        check(lib().xtb_muzero_replay_add(self.handle, model.handle if values is None else None, slot, off, e0, ne, p[0], p[1], p[2],
                                          p[3], p[4], L, p[5] if values is not None else None, stream_ptr()))
        self.planner.commit(placement, L)     # only a stored trajectory moves the planner
        if ne and not self._warned:
            self._warned = True
            warnings.warn("MuZero device replay: DEVICE_REPLAY_STEPS is full, the oldest trajectories are evicted before the "
                          "ring overwrites them; draws now differ from the host buffer's", RuntimeWarning)
        return slot

    def buffers(self, B):
        """Device buffers of a B-sample step: uniforms [2B] float64, slot / pos [B] int32, the gathered batch, and the
        loss (float32) and status (int32) side by side for one download."""
        b = self._bufs.get(B)
        if b is None:
            dev, K = self.device, self.K
            out = torch.zeros(2, dtype=torch.float32, device=dev)
            b = dict(u=torch.empty(2 * B, dtype=torch.float64, device=dev), slot=torch.empty(B, dtype=torch.int32, device=dev),
                     pos=torch.empty(B, dtype=torch.int32, device=dev),
                     obs=torch.empty((B,) + self.obs_shape, dtype=torch.uint8 if self.obs_dtype.itemsize == 1 else torch.float32,
                                     device=dev),
                     action=torch.empty(B, K, dtype=torch.int32, device=dev), tv=torch.empty(B, K + 1, dtype=torch.float32, device=dev),
                     tr=torch.empty(B, K + 1, dtype=torch.float32, device=dev),
                     tp=torch.empty(B, K + 1, self.A, dtype=torch.float32, device=dev),
                     values=torch.empty(B, dtype=torch.float64, device=dev), out=out, loss=out[:1], status=out[1:].view(torch.int32))
            bt = capi.MuzeroReplayBatch()
            bt.obs, bt.action, bt.target_value = b["obs"].data_ptr(), b["action"].data_ptr(), b["tv"].data_ptr()
            bt.target_reward, bt.target_policy = b["tr"].data_ptr(), b["tp"].data_ptr()
            b["batch"] = bt
            self._bufs[B] = b
        return b

    def sample(self, uniforms):
        """The draw from 2B host uniforms (B trajectory uniforms, then B position uniforms) -> (slot, pos, the gathered
        batch obs / action / tv / tr / tp), device tensors overwritten by the next call of the same size."""
        B = len(uniforms) // 2
        b = self.buffers(B)
        stage_h2d(b["u"], np.asarray(uniforms, np.float64), np.float64)
        check(lib().xtb_muzero_replay_sample(self.handle, B, _ptr(b["u"]), _ptr(b["slot"]), _ptr(b["pos"]), C.byref(b["batch"]),
                                             stream_ptr()))
        return b["slot"], b["pos"], b["obs"], b["action"], b["tv"], b["tr"], b["tp"]

    def update(self, slot, pos, values):
        """The priority updates of one step from its post-step values [B] (host float64) -> the status bits."""
        B = len(values)
        b = self.buffers(B)
        stage_h2d(b["values"], np.asarray(values, np.float64), np.float64)
        check(lib().xtb_muzero_replay_update(self.handle, B, _ptr(slot), _ptr(pos), _ptr(b["values"]), stream_ptr()))
        return self.status()

    def status(self):
        """The status bits (capi.MZR_*) of the last draw and the updates after it, without the rest of the state."""
        st = C.c_int()
        check(lib().xtb_muzero_replay_state(self.handle, None, C.byref(st), None, None, None, None))
        return st.value

    def train(self, model, uniforms):
        """One learner step as one call (xtb_muzero_replay_train, graph-replayed when the model uses graphs): one staged
        upload of the uniforms, one download of the loss and the status -> (loss, status)."""
        B = len(uniforms) // 2
        model._check_batch(B)
        b = self.buffers(B)
        stage_h2d(b["u"], np.asarray(uniforms, np.float64), np.float64)
        check(lib().xtb_muzero_replay_train(self.handle, model.handle, model.opt.handle, B, _ptr(b["u"]), _ptr(b["slot"]), _ptr(b["pos"]),
                                            C.byref(b["batch"]), float(model.weight_decay_loss), _ptr(b["loss"]), _ptr(b["status"]),
                                            1 if model.use_graph else 0, stream_ptr()))
        out = b["out"].cpu().numpy()
        return float(out[0]), int(out[1:].view(np.int32)[0])

    def state(self):
        """Snapshot: count, status, the slot table (off, len, live arrays), the trajectory tree and the forest."""
        cnt, status, leaves = C.c_int(), C.c_int(), C.c_int()
        check(lib().xtb_muzero_replay_state(self.handle, C.byref(cnt), C.byref(status), C.byref(leaves), None, None, None))
        slots = (capi.MuzeroReplaySlot * self.planner.size)()
        tree = np.zeros(2 * leaves.value, np.float64)
        forest = np.zeros(4 * self.planner.steps, np.float64)
        check(lib().xtb_muzero_replay_state(self.handle, None, None, None, slots, tree.ctypes.data, forest.ctypes.data))
        return dict(count=cnt.value, status=status.value, leaves=leaves.value, off=np.array([s.off for s in slots]),
                    len=np.array([s.len for s in slots]), live=np.array([s.live for s in slots], bool), traj_tree=tree, forest=forest)

    def position_leaves(self, st, slot):
        """The position priorities of `slot` in a state() snapshot."""
        off, L = int(st["off"][slot]), int(st["len"][slot])
        cap = 1
        while cap < L:
            cap *= 2
        return st["forest"][4 * off + cap:4 * off + cap + L - self.K]


def _device_replay_config(alg_config):
    """DEVICE_REPLAY (bool, default False) and DEVICE_REPLAY_STEPS (positive int), checked before anything touches CUDA."""
    cfg = alg_config or {}
    on, steps = cfg.get("DEVICE_REPLAY", False), cfg.get("DEVICE_REPLAY_STEPS", _DEFAULT_REPLAY_STEPS)
    if not isinstance(on, (bool, np.bool_)):
        raise ValueError("DEVICE_REPLAY must be a bool, got {!r}".format(on))
    if isinstance(steps, (bool, np.bool_)) or not isinstance(steps, numbers.Integral) or steps < 1:
        raise ValueError("DEVICE_REPLAY_STEPS must be a positive int, got {!r}".format(steps))
    return bool(on), int(steps)


@Registers.algorithm
class Muzero(Algorithm):
    """Muzero learner: prepare_data stores trajectories, train samples and runs one MuzeroModel step.

    alg_config DEVICE_REPLAY True keeps the replay on the device (DeviceTrajectoryReplay over DEVICE_REPLAY_STEPS pool
    steps): prepare_data uploads each trajectory once and builds its priorities there, and train() is one staged upload
    of the host's 2 BATCH_SIZE uniforms, one graph (draw, gather, model step, priority updates) and one download."""

    device_replay = False

    def __init__(self, model_info, alg_config, **kwargs):
        device_replay, replay_steps = _device_replay_config(alg_config)
        import_config(globals(), alg_config)
        super().__init__(alg_name=kwargs.get("name") or "muzero", model_info=model_info["actor"], alg_config=alg_config)
        self.discount = GAMMA
        self.unroll_step = UNROLL_STEP
        self.td_step = TD_STEP
        self.batch_size = BATCH_SIZE
        self.async_flag = False
        if getattr(self.actor, "td_step", UNROLL_STEP) != UNROLL_STEP:
            raise ValueError("UNROLL_STEP {} != the model's td_step {}".format(UNROLL_STEP, self.actor.td_step))
        self.device_replay = device_replay
        if device_replay:
            a = self.actor
            self.buff = DeviceTrajectoryReplay(BUFFER_SIZE, replay_steps, a.state_dim, a._np_dt, a.action_dim, UNROLL_STEP,
                                               max(a.max_batch, BATCH_SIZE), a.device)
        else:
            self.buff = PrioritizedBuffer(BUFFER_SIZE, alpha=1)

    def prepare_data(self, train_data, **kwargs):
        """muzero.py:88-97: keep trajectories longer than UNROLL_STEP + 1, priority per position |value - target|."""
        K = self.unroll_step
        if self.device_replay:
            if len(train_data["reward"]) > K + 1:
                self.buff.add(train_data, model=self.actor)
            return
        if len(train_data["reward"]) > K + 1:
            value = self.actor.value_inference(np.asarray(train_data["cur_state"]))
            pri = np.abs(value - np.asarray(train_data["target_value"]))
            pos_buff = PrioritizedBuffer(len(pri), alpha=1)
            for i in range(len(pri) - K):
                pos_buff.add(0, pri[i])
            train_data.update({"pos_buff": pos_buff})
            self.buff.add(train_data, pos_buff.weight())

    def sample_batch(self):
        """The trajectories and positions of one training batch and the gathered minibatch (muzero.py:52-79)."""
        K = self.unroll_step
        trajs, _, _ = self.buff.sample(self.batch_size, 1)
        pos = [t["pos_buff"].sample(1, 1)[2][0] for t in trajs]
        image = np.stack([np.asarray(t["cur_state"][i]) for t, i in zip(trajs, pos)])
        actions = np.stack([np.asarray(t["action"][i:i + K]) for t, i in zip(trajs, pos)]).astype(np.int32)
        tv = np.array([[t["target_value"][j] for j in range(i, i + K + 1)] for t, i in zip(trajs, pos)], np.float64)
        tr = np.array([[t["reward"][j] for j in range(i, i + K + 1)] for t, i in zip(trajs, pos)], np.float64)
        tp = np.array([[t["child_visits"][j] for j in range(i, i + K + 1)] for t, i in zip(trajs, pos)], np.float64)
        return trajs, pos, image, actions, tv, tr, tp

    def train(self, **kwargs):
        """muzero.py:50-86: 0 until BATCH_SIZE trajectories are stored; else one step, then the new priorities."""
        if len(self.buff) < self.batch_size:
            return 0
        if self.device_replay:
            u = [random.random() for _ in range(2 * self.batch_size)]   # the host's draws, in its order
            loss, status = self.buff.train(self.actor, u)
            if status & capi.MZR_BAD_PRIORITY:
                raise ValueError("a priority update met a priority that is not > 0; the updates stopped there")
            if status & capi.MZR_BAD_INDEX:
                raise ValueError("a priority update named no stored trajectory or position; the updates stopped there")
            return loss
        trajs, pos, image, actions, tv, tr, tp = self.sample_batch()
        loss, value = self.actor.train_and_values(image, actions, tv, tr, tp)
        new_pri = np.maximum(np.abs(value - tv[:, 0]), 1e-5)
        for i, (t, p) in enumerate(zip(trajs, pos)):
            t["pos_buff"].update_priorities([p], [new_pri[i]])
            # the reference writes the trajectory's new weight at the BATCH position i, not at the sampled index
            self.buff.update_priorities([i], [t["pos_buff"].weight()])
        return loss
