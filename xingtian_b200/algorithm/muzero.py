"""The Muzero learner (xt/algorithm/muzero/muzero.py) over MuzeroCnn / MuzeroMlp.

Trajectories live on the host in a proportional prioritised buffer (segment trees written for this package with the query
semantics the reference's learner relies on); each training call samples BATCH_SIZE trajectories and one position per
trajectory, gathers the observation, the UNROLL_STEP actions and the UNROLL_STEP + 1 targets of every sample, uploads the
minibatch through the staged pinned copy and runs one model step, which also returns the post-update values used as
the new priorities."""
import operator
import random

import numpy as np

from ..registry import Registers, import_config
from .base import Algorithm

# xt/algorithm/muzero/default_config.py
BATCH_SIZE = 1024
BUFFER_SIZE = 100000
GAMMA = 0.997
TD_STEP = 10
UNROLL_STEP = 5


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


@Registers.algorithm
class Muzero(Algorithm):
    """Muzero learner: prepare_data stores trajectories, train samples and runs one MuzeroModel step."""

    def __init__(self, model_info, alg_config, **kwargs):
        import_config(globals(), alg_config)
        super().__init__(alg_name=kwargs.get("name") or "muzero", model_info=model_info["actor"], alg_config=alg_config)
        self.buff = PrioritizedBuffer(BUFFER_SIZE, alpha=1)
        self.discount = GAMMA
        self.unroll_step = UNROLL_STEP
        self.td_step = TD_STEP
        self.batch_size = BATCH_SIZE
        self.async_flag = False
        if getattr(self.actor, "td_step", UNROLL_STEP) != UNROLL_STEP:
            raise ValueError("UNROLL_STEP {} != the model's td_step {}".format(UNROLL_STEP, self.actor.td_step))

    def prepare_data(self, train_data, **kwargs):
        """muzero.py:88-97: keep trajectories longer than UNROLL_STEP + 1, priority per position |value - target|."""
        K = self.unroll_step
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
        trajs, pos, image, actions, tv, tr, tp = self.sample_batch()
        loss, value = self.actor.train_and_values(image, actions, tv, tr, tp)
        new_pri = np.maximum(np.abs(value - tv[:, 0]), 1e-5)
        for i, (t, p) in enumerate(zip(trajs, pos)):
            t["pos_buff"].update_priorities([p], [new_pri[i]])
            # the reference writes the trajectory's new weight at the BATCH position i, not at the sampled index
            self.buff.update_priorities([i], [t["pos_buff"].weight()])
        return loss
