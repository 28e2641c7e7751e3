"""Replay buffers: the reference's host deque (xt/algorithm/replay_buffer.py:24-42) and a
device-resident ring used by the fused DQN step."""
import ctypes as C
import random
from collections import deque

import numpy as np
import torch

from ..capi import check, lib
from ..engine import stream_ptr


class ReplayBuffer(object):
    """xt/algorithm/replay_buffer.py:24-42 (uniform sampling without replacement)."""

    def __init__(self, buffer_size):
        self.buffer = deque(maxlen=buffer_size)

    def get_batch(self, batch_size):
        sample_size = min(self.size(), batch_size)
        return random.sample(self.buffer, int(sample_size))

    def size(self):
        return len(self.buffer)

    def add(self, train_data):
        self.buffer.append(train_data)


class DeviceReplayBuffer(object):
    """Ring of transitions in HBM: frames are stored once per transition slot as (s, s') uint8
    pairs like the reference deque (56 KB / transition at 84x84x4); sampling draws the same
    `random.sample(range(size), k)` indices on the host and gathers on the device.

    `prioritized` = (alpha, eps, seed): the ring also owns a native sum / min tree over its slots (xtb_per, leaf i = slot
    i) that every written slot enters at the largest priority so far; the prioritized DQN step samples and updates it
    on the device."""

    def __init__(self, buffer_size, state_dim, obs_dtype, device, prioritized=None):
        self.capacity = int(buffer_size)
        self.per = None
        if prioritized is not None:
            alpha, eps, seed = prioritized
            h = C.c_void_p()
            check(lib().xtb_per_create(self.capacity, float(alpha), float(eps), int(seed), C.byref(h)))
            self.per = h
        self.device = device
        self.state_dim = tuple(state_dim)
        self.obs_dtype = obs_dtype
        self._alloc = 0
        self.count = 0      # valid entries
        self.head = 0       # next write slot
        self.obs = self.next_obs = self.action = self.reward = self.done = self.disc = None
        self.keep_disc = False   # n-step replay: per-transition bootstrap discount

    def _grow(self, need):
        if need <= self._alloc:
            return
        new = min(self.capacity, max(need, 1024, self._alloc * 2))
        def mk(shape, dt, old):
            t = torch.empty(shape, dtype=dt, device=self.device)
            if old is not None:
                t[:self._alloc].copy_(old)
            return t
        self.obs = mk((new,) + self.state_dim, self.obs_dtype, self.obs)
        self.next_obs = mk((new,) + self.state_dim, self.obs_dtype, self.next_obs)
        self.action = mk((new,), torch.int32, self.action)
        self.reward = mk((new,), torch.float32, self.reward)
        self.done = mk((new,), torch.uint8, self.done)
        if self.keep_disc:
            self.disc = mk((new,), torch.float32, self.disc)
        self._alloc = new

    def __del__(self):
        try:
            if getattr(self, "per", None) is not None:
                lib().xtb_per_destroy(self.per)
                self.per = None
        except Exception:  # interpreter shutdown
            pass

    def size(self):
        return self.count

    def add_batch(self, obs, action, reward, next_obs, done, disc=None):
        """Arrays may be numpy (host) or torch tensors already on the device."""
        n = len(action)
        np_dt = np.uint8 if self.obs_dtype == torch.uint8 else np.float32
        def up(x, dt, flat=True):
            if torch.is_tensor(x):
                return x.to(self.device).reshape(-1) if flat else x.to(self.device)
            a = np.ascontiguousarray(x, dt)
            return torch.from_numpy(a.reshape(-1) if flat else a).to(self.device, non_blocking=not flat)
        obs = up(obs, np_dt, flat=False)
        nxt = up(next_obs, np_dt, flat=False)
        act = up(action, np.int32)
        rew = up(reward, np.float32)
        don = done.reshape(-1) if torch.is_tensor(done) else torch.from_numpy(np.ascontiguousarray(done, np.bool_).reshape(-1).view(np.uint8)).to(self.device)
        dsc = up(disc, np.float32) if disc is not None else None
        done_n = 0
        while done_n < n:
            self._grow(min(self.capacity, self.head + (n - done_n)))
            k = min(n - done_n, self._alloc - self.head)
            sl = slice(self.head, self.head + k)
            src = slice(done_n, done_n + k)
            self.obs[sl].copy_(obs[src]); self.next_obs[sl].copy_(nxt[src])
            self.action[sl].copy_(act[src]); self.reward[sl].copy_(rew[src]); self.done[sl].copy_(don[src])
            if self.keep_disc and dsc is not None:
                self.disc[sl].copy_(dsc[src])
            if self.per is not None:
                check(lib().xtb_per_add(self.per, self.head, k, stream_ptr()))
            self.head = (self.head + k) % self.capacity
            self.count = min(self.capacity, self.count + k)
            done_n += k

    def sample_indices(self, batch_size):
        """Same draw as ReplayBuffer.get_batch: random.sample over the live entries (oldest first)."""
        k = min(self.count, batch_size)
        picks = random.sample(range(self.count), int(k))
        if self.count == self.capacity:   # logical index 0 = oldest = head
            picks = [(self.head + p) % self.capacity for p in picks]
        return np.asarray(picks, np.int64)

    def gather(self, idx):
        idx = torch.from_numpy(idx).to(self.device)
        return (self.obs.index_select(0, idx), self.action.index_select(0, idx), self.reward.index_select(0, idx),
                self.next_obs.index_select(0, idx), self.done.index_select(0, idx))
