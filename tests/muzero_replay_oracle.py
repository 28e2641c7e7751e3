"""Host restatement of the Muzero learner's device replay (DeviceTrajectoryReplay, xtb_muzero_replay in xtb200.h), built
on the host learner's PrioritizedBuffer: PoolPlanner places every trajectory; an evicted slot's leaf becomes 0, a
batch-position write never revives it, and a descent that ends on a slot without a live trajectory takes the nearest
live slot below it, wrapping from slot 0 to the newest.  Without evictions it is the host learner itself."""
import numpy as np

from xingtian_b200.algorithm.muzero import PoolPlanner, PrioritizedBuffer


class RestatedReplay(object):
    def __init__(self, size, steps, unroll):
        self.buff = PrioritizedBuffer(size, alpha=1)
        self.planner = PoolPlanner(size, steps)
        self.K = unroll

    def __len__(self):
        return len(self.buff)

    def add(self, traj, values):
        """Muzero.prepare_data with the given position values -> the slot."""
        L = len(traj["reward"])
        pri = np.abs(np.asarray(values, np.float64) - np.asarray(traj["target_value"], np.float64))
        pos_buff = PrioritizedBuffer(L, alpha=1)
        for i in range(L - self.K):
            pos_buff.add(0, pri[i])
        slot, _, e0, ne = self.planner.place(L)
        assert self.buff.add(dict(traj, pos_buff=pos_buff), pos_buff.weight()) == slot
        for k in range(ne):
            self.buff._set((e0 + k) % self.buff.size, 0.0)
        return slot

    def draw(self, u):
        """The draw from the 2B uniforms the host learner would take -> (slots, positions)."""
        B, n, live = len(u) // 2, len(self.buff), self.planner.live
        step = self.buff.it_sum.reduce(0, n - 1) / B
        slots = []
        for k in range(B):
            j = self.buff.it_sum.find_prefixsum_idx(u[k] * step + k * step)
            if j >= n or not live[j]:
                start = min(j, n)
                j = next(c for c in ((start - q) % n for q in range(1, n + 1)) if live[c])
            slots.append(j)
        pos = []
        for k, s in enumerate(slots):
            pb = self.buff.storage[s]["pos_buff"]
            tot = pb.it_sum.reduce(0, len(pb) - 1)
            pos.append(min(pb.it_sum.find_prefixsum_idx(u[B + k] * tot + 0 * tot), len(pb) - 1))
        return slots, pos

    def gather(self, slots, pos):
        K, st = self.K, self.buff.storage
        image = np.stack([np.asarray(st[s]["cur_state"][p]) for s, p in zip(slots, pos)])
        actions = np.stack([np.asarray(st[s]["action"][p:p + K]) for s, p in zip(slots, pos)]).astype(np.int32)
        tv = np.array([st[s]["target_value"][p:p + K + 1] for s, p in zip(slots, pos)], np.float64)
        tr = np.array([st[s]["reward"][p:p + K + 1] for s, p in zip(slots, pos)], np.float64)
        tp = np.array([st[s]["child_visits"][p:p + K + 1] for s, p in zip(slots, pos)], np.float64)
        return image, actions, tv, tr, tp

    def update(self, slots, pos, values):
        """Muzero.train's updates from the post-step values, batch position by batch position."""
        tv = np.array([self.buff.storage[s]["target_value"][p] for s, p in zip(slots, pos)], np.float64)
        new_pri = np.maximum(np.abs(np.asarray(values, np.float64) - tv), 1e-5)
        for i, (s, p) in enumerate(zip(slots, pos)):
            pb = self.buff.storage[s]["pos_buff"]
            pb.update_priorities([p], [new_pri[i]])
            if self.planner.live[i]:
                self.buff.update_priorities([i], [pb.weight()])

    def traj_leaves(self):
        return np.array([self.buff.it_sum[i] for i in range(len(self.buff))])

    def pos_leaves(self, slot):
        pb = self.buff.storage[slot]["pos_buff"]
        return np.array([pb.it_sum[i] for i in range(len(pb))])
