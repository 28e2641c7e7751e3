"""IMPALAOpt algorithm (xt/algorithm/impala/impala_opt.py:37-147)."""
import os

import numpy as np
import torch

from ..engine import DeviceStore, stage_h2d
from ..registry import Registers, import_config
from .base import Algorithm, FIFODistPolicy

BATCH_SIZE = 200   # xt/algorithm/impala/default_config.py


@Registers.algorithm
class IMPALAOpt(Algorithm):
    """Buffers (state, behaviour logits, action, done, reward) trajectories on the device and trains
    in BATCH_SIZE slices; V-trace runs inside the train step."""

    def __init__(self, model_info, alg_config, **kwargs):
        import_config(globals(), alg_config)
        super().__init__(alg_name="impala", model_info=model_info["actor"], alg_config=alg_config)
        m = self.actor
        # grow-only device trajectory store: its addresses stay put between iterations, so the captured train-step graphs
        # (keyed by their buffers) are replayed instead of re-captured
        self._store = DeviceStore(m.device, obs=(tuple(m.state_dim), torch.uint8), bp=((m.action_dim,), torch.float32),
                                  action=((), torch.int32), done=((), torch.uint8), reward=((), torch.float32))
        self._losses, self._tmp = None, None
        self.async_flag = False
        self.dist_model_policy = FIFODistPolicy(alg_config["instance_num"], prepare_times=self._prepare_times_per_train)

    @staticmethod
    def _data_proc(episode_data):
        """impala_opt.py:125-147."""
        states = episode_data["cur_state"]
        behavior_logits = episode_data["logit"]
        actions = episode_data["action"]
        dones = np.asarray(episode_data["done"], dtype=np.bool_)
        rewards = np.asarray(episode_data["reward"])
        return states, behavior_logits, actions, dones, rewards

    def prepare_data(self, train_data, **kwargs):
        """impala_opt.py:110-117 -- staged straight into the device store (pinned ring, asynchronous)."""
        state, logit, action, done, reward = self._data_proc(train_data)
        n, st = len(state), self._store
        st.reserve(st.n + n)
        sl = slice(st.n, st.n + n)
        stage_h2d(st.obs[sl], state, np.uint8)
        stage_h2d(st.bp[sl], logit, np.float32)
        stage_h2d(st.action[sl], np.asarray(action).reshape(-1), np.int32)
        stage_h2d(st.done[sl], np.ascontiguousarray(done, np.bool_).reshape(-1).view(np.uint8), np.uint8)
        stage_h2d(st.reward[sl], np.asarray(reward).reshape(-1), np.float32)
        st.n += n

    def train(self, **kwargs):
        """impala_opt.py:73-106: concatenate, slice by BATCH_SIZE, one SGD step per slice, mean loss."""
        cat, nbatch = self._store, self._store.n
        if nbatch == 0:
            raise ValueError("need at least one array to concatenate")
        count = (nbatch + BATCH_SIZE - 1) // BATCH_SIZE
        if self._losses is None or self._losses.numel() < count:
            self._losses = torch.zeros(count, dtype=torch.float32, device=self.actor.device)
            self._tmp = torch.zeros(1, dtype=torch.float32, device=self.actor.device)
        losses, tmp = self._losses[:count], self._tmp
        for i in range(count):
            s, e = i * BATCH_SIZE, min(nbatch, (i + 1) * BATCH_SIZE)
            self.actor.train_device(cat.obs[s:e], cat.bp[s:e], cat.action[s:e], cat.done[s:e], cat.reward[s:e], e - s, tmp)
            losses[i:i + 1].copy_(tmp)
        cat.n = 0
        return float(losses.mean().cpu())

    def save(self, model_path, model_index):
        """impala_opt.py:103-108."""
        actor_name = "actor" + str(model_index).zfill(5)
        actor_name = self.actor.save_model(os.path.join(model_path, actor_name))
        return [actor_name.split("/")[-1]]

    def predict(self, state):
        """impala_opt.py:119-123."""
        return self.actor.predict(state)
