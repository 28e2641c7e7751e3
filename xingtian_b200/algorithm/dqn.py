"""DQN algorithm (xt/algorithm/dqn/dqn.py:36-148)."""
import math
import numbers

import numpy as np
import torch

from ..capi import PER_NONFINITE
from ..registry import Registers, import_config, model_builder
from .base import Algorithm
from .replay_buffer import DeviceReplayBuffer

# xt/algorithm/dqn/default_config.py
BATCH_SIZE = 32
BUFFER_SIZE = 100000
TARGET_UPDATE_FREQ = 1000
GAMMA = 0.99
# extensions named by BASELINE.json's north_star; the defaults are the reference (1-step TD, Keras 'mse')
N_STEP = 1
HUBER_DELTA = 0.0
# prioritized replay (Schaul et al., proportional; the rules of xt/algorithm/prioritized_replay_buffer_muzero.py), off by
# default; beta stays constant
PRIORITIZED_REPLAY = False
PRIORITY_ALPHA = 0.6
PRIORITY_BETA = 0.4
PRIORITY_EPS = 1e-6


def priority_config(alg_config):
    """(on, alpha, beta, eps) from alg_config, each key also accepted in lower case, the module defaults otherwise.
    Raises ValueError for a value the device sampler rejects (alpha < 0, beta <= 0, eps <= 0, not finite, a flag that is
    not a bool)."""
    def get(key):
        return alg_config.get(key, alg_config.get(key.lower(), globals()[key]))
    on = get("PRIORITIZED_REPLAY")
    if not isinstance(on, (bool, np.bool_)):
        raise ValueError("DQN: prioritized_replay must be True or False, got %r" % (on,))
    vals = {}
    for key, low in (("PRIORITY_ALPHA", 0.0), ("PRIORITY_BETA", None), ("PRIORITY_EPS", None)):
        v = get(key)
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or \
                (v < low if low is not None else not v > 0):
            raise ValueError("DQN: %s must be a finite number %s, got %r" % (key, ">= 0" if low is not None else "> 0", v))
        vals[key] = float(v)
    return bool(on), vals["PRIORITY_ALPHA"], vals["PRIORITY_BETA"], vals["PRIORITY_EPS"]


@Registers.algorithm
class DQN(Algorithm):
    """Online + target network, device replay ring, fused TD-target/mse/Adam step."""

    def __init__(self, model_info, alg_config, **kwargs):
        per, alpha, beta, eps = priority_config(alg_config)     # before anything is built on the device
        import_config(globals(), alg_config)
        model_info = model_info["actor"]
        super().__init__(alg_name="dqn", model_info=model_info, alg_config=alg_config)
        self.target_actor = model_builder(model_info)
        self.update_target()     # keras builds the target with its own init; synced at first update in the
        # reference -- here both start equal, which only changes the first TARGET_UPDATE_FREQ steps
        obs_dt = torch.uint8 if self.actor.arch["input_dtype"] == "uint8" else torch.float32
        self.prioritized, self.priority_beta = per, beta
        # the Philox seed of the device draws: one global np.random draw, as the models' sampling seeds
        prio = (alpha, eps, int(np.random.randint(0, 2 ** 31 - 1))) if per else None
        self.buff = DeviceReplayBuffer(BUFFER_SIZE, self.actor.state_dim, obs_dt, self.actor.device, prioritized=prio)
        self.double_dqn = alg_config.get("double_dqn", False)
        self.n_step = int(alg_config.get("N_STEP", alg_config.get("n_step", N_STEP)))
        self.huber_delta = float(alg_config.get("HUBER_DELTA", alg_config.get("huber_delta", HUBER_DELTA)))
        self.buff.keep_disc = self.n_step > 1
        self._loss = torch.zeros(1, dtype=torch.float32, device=self.actor.device)
        self._idx_dev = None
        if per:
            dev = self.actor.device
            self._per_idx = torch.zeros(BATCH_SIZE, dtype=torch.int32, device=dev)
            self._per_w = torch.zeros(BATCH_SIZE, dtype=torch.float32, device=dev)
            self._per_td = torch.zeros(BATCH_SIZE, dtype=torch.float32, device=dev)
            self._per_status = torch.zeros(1, dtype=torch.int32, device=dev)

    def train(self, **kwargs):
        """dqn.py:61-103."""
        if self.prioritized:
            return self.train_prioritized()
        idx = self.buff.sample_indices(BATCH_SIZE)
        loss = self.train_on_indices(idx)
        return loss

    def train_prioritized(self):
        """One step over BATCH_SIZE rows drawn from the priority tree, as one device graph: stratified draw with importance
        weights, the weighted TD step, and the rows' new priorities (|TD error| + eps) ** alpha.  Returns the weighted
        loss; raises FloatingPointError once an update has met a priority that is not finite."""
        b = self.buff
        if b.count == 0:
            raise RuntimeError("DQN.train: the replay buffer is empty")
        self.actor.train_per_device(self.target_actor, b.per, self.priority_beta, b.obs, b.action, b.reward, b.next_obs, b.done,
                                    BATCH_SIZE, GAMMA, self._loss, self._per_idx, self._per_w, self._per_td, self._per_status,
                                    double_dqn=self.double_dqn, disc=b.disc if self.n_step > 1 else None,
                                    huber_delta=self.huber_delta)
        loss = float(self._loss.cpu()[0])
        status = int(self._per_status.cpu()[0])
        if status & PER_NONFINITE:
            raise FloatingPointError("DQN.train: a TD error gave a priority that is not finite (loss %r)" % loss)
        if status:
            raise RuntimeError("DQN.train: prioritized replay status %d" % status)
        return self._after_step(loss)

    def train_on_indices(self, idx):
        """One SGD step on replay rows `idx`: the native step gathers the rows of the ring itself (no batch copy)."""
        n = int(len(idx))
        if self._idx_dev is None or self._idx_dev.numel() < n:
            self._idx_dev = torch.empty(max(n, BATCH_SIZE), dtype=torch.int32, device=self.actor.device)
        self._idx_dev[:n].copy_(torch.from_numpy(np.ascontiguousarray(idx, np.int32)))
        b = self.buff
        self.actor.train_td_device(self.target_actor, b.obs, b.action, b.reward, b.next_obs, b.done, n, GAMMA, self._loss,
                                   double_dqn=self.double_dqn, idx=self._idx_dev, disc=b.disc if self.n_step > 1 else None,
                                   huber_delta=self.huber_delta)
        return self._after_step(float(self._loss.cpu()[0]))

    def _after_step(self, loss):
        self.train_count += 1
        if self.train_count % TARGET_UPDATE_FREQ == 0:
            self.update_target()
        return loss

    def restore(self, model_name=None, model_weights=None):
        """dqn.py:105-119."""
        if model_weights is not None:
            self.actor.set_weights(model_weights)
            self.target_actor.set_weights(model_weights)
        else:
            self.actor.load_model(model_name)
            self.target_actor.load_model(model_name)

    def prepare_data(self, train_data, **kwargs):
        """dqn.py:121-138.  With N_STEP > 1 the incoming trajectory segment is rewritten into n-step transitions on the
        device (xtb_nstep_returns): reward = n-step return, next_state = state after the window, done = window hit a
        terminal, plus the bootstrap discount gamma^m."""
        cur, act = np.asarray(train_data["cur_state"]), np.asarray(train_data["action"])
        rew, nxt, done = np.asarray(train_data["reward"]), np.asarray(train_data["next_state"]), np.asarray(train_data["done"])
        if self.n_step <= 1:
            self.buff.add_batch(cur, act, rew, nxt, done)
            return
        import ctypes as C
        from ..engine import _ptr, stream_ptr
        from ..capi import check, lib
        dev = self.actor.device
        T = len(act)
        r_d = torch.from_numpy(np.ascontiguousarray(rew, np.float32).reshape(-1)).to(dev)
        d_d = torch.from_numpy(np.ascontiguousarray(done, np.bool_).reshape(-1).view(np.uint8)).to(dev)
        ret = torch.empty(T, dtype=torch.float32, device=dev); disc = torch.empty_like(ret)
        last = torch.empty(T, dtype=torch.int32, device=dev); dn = torch.empty(T, dtype=torch.uint8, device=dev)
        check(lib().xtb_nstep_returns(_ptr(r_d), _ptr(d_d), 1, T, self.n_step, float(GAMMA), _ptr(ret), _ptr(disc), _ptr(last),
                                      _ptr(dn), stream_ptr()))
        np_dt = np.uint8 if self.buff.obs_dtype == torch.uint8 else np.float32
        nxt_d = torch.from_numpy(np.ascontiguousarray(nxt, np_dt)).to(dev).index_select(0, last.long())
        self.buff.add_batch(cur, act, ret, nxt_d, dn, disc=disc)

    def update_target(self):
        """dqn.py:140-148: hard copy (device to device)."""
        self.target_actor.net.load_flat(self.actor.net.params)
