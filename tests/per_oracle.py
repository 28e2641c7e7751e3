"""Float64 restatement of prioritized replay over the slots of a device ring (xtb_per, include/xtb200.h): the reference's
PrioritizedReplayBuffer rules (xt/algorithm/prioritized_replay_buffer_muzero.py:77-200) with leaf i = ring slot i, the
total taken over every stored leaf, and a draw past the stored slots clamped to count - 1."""
import math

import numpy as np


def leaf_count(capacity):
    leaves = 1
    while leaves < capacity:
        leaves *= 2
    return leaves


class PerTree(object):
    """Sum and min trees in heap order (node 1 the root, node i's children 2i and 2i + 1, leaf j at node leaves + j),
    every internal node op(left, right) of its children."""

    def __init__(self, capacity, alpha, eps):
        self.leaves = leaf_count(capacity)
        self.alpha, self.eps = alpha, eps
        self.sum = np.zeros(2 * self.leaves)
        self.mn = np.full(2 * self.leaves, np.inf)
        self.count, self.max_priority = 0, 1.0

    def _rebuild(self):
        for node in range(self.leaves - 1, 0, -1):
            self.sum[node] = self.sum[2 * node] + self.sum[2 * node + 1]
            self.mn[node] = min(self.mn[2 * node], self.mn[2 * node + 1])

    def add(self, first, n):
        """ring slots [first, first + n) were written: each enters at max_priority ** alpha"""
        p = self.max_priority ** self.alpha
        self.sum[self.leaves + first:self.leaves + first + n] = p
        self.mn[self.leaves + first:self.leaves + first + n] = p
        self.count = max(self.count, first + n)
        self._rebuild()

    def update(self, idx, td_abs):
        """update_priorities' sequential loop on priorities |delta| + eps (float32 |delta|); a priority that is not finite
        is skipped.  Returns True when one was."""
        bad = False
        for j, t in zip(idx, np.asarray(td_abs, np.float32)):
            d = float(t) + self.eps
            if not math.isfinite(d) or not math.isfinite(d ** self.alpha):
                bad = True
                continue
            self.sum[self.leaves + j] = self.mn[self.leaves + j] = d ** self.alpha
            self.max_priority = max(self.max_priority, d)
        self._rebuild()
        return bad


def descend(sum_tree, leaves, count, u):
    """Stratified draw of B = len(u) leaves: mass_k = (u_k + k) total / B, the first leaf whose running sum exceeds it,
    clamped to count - 1."""
    total, B = float(sum_tree[1]), len(u)
    out = np.empty(B, np.int64)
    for k in range(B):
        mass = (float(u[k]) + k) * total / B
        node = 1
        while node < leaves:
            left = float(sum_tree[2 * node])
            if left > mass:
                node = 2 * node
            else:
                mass -= left
                node = 2 * node + 1
        out[k] = min(node - leaves, count - 1)
    return out


def weights(sum_tree, min_tree, leaves, count, idx, beta):
    """w_k = ((leaf / total) count) ** -beta / (p_min count) ** -beta, p_min = max(min / total, 1e-5), float64"""
    total = float(sum_tree[1])
    p_min = max(float(min_tree[1]) / total, 1e-5)
    max_w = (p_min * count) ** (-beta)
    return np.array([((float(sum_tree[leaves + j]) / total) * count) ** (-beta) / max_w for j in idx])
