"""PPO algorithm on the device rollout store (xt/algorithm/ppo/ppo.py:30-95)."""
import logging

import numpy as np
import torch

from ..capi import check
from ..engine import DeviceStore, _ptr, stage_h2d, stream_ptr
from ..registry import Registers, import_config
from .base import Algorithm

GAMMA, LAM = 0.99, 0.95   # xt/agent/ppo/default_config.py:2-3 (the agent imports them by value)


@Registers.algorithm
class PPO(Algorithm):
    """Accumulates trajectories straight into HBM (pinned staging + async H2D per trajectory) instead
    of python lists + np.concatenate, then runs the fused minibatch-SGD loop.

    ``prepare_data`` accepts the reference trajectory dict (xt/agent/ppo/ppo.py:99-106: cur_state,
    action, logp, adv, old_value, target_value) and also the *raw* form (value[T+1], reward, done
    instead of adv/target_value): then GAE (agent/ppo/ppo.py:77-106) runs on the device."""

    def __init__(self, model_info, alg_config, **kwargs):
        import_config(globals(), alg_config)
        super().__init__(alg_name=kwargs.get("name") or "ppo", model_info=model_info["actor"], alg_config=alg_config)
        # raw trajectories: reward / done at their rollout rows, value[T+1] per trajectory back to back
        dev = self.actor.device
        self._raw_steps = DeviceStore(dev, rew=((), torch.float32), don=((), torch.uint8))
        self._raw_values = DeviceStore(dev, val=((), torch.float32))
        self._init_train_list()
        self.async_flag = False
        self.sign_clip_reward = bool(alg_config.get("sign_clip_reward", False))
        if model_info.get("finetune_weight"):
            self.actor.load_model(model_info["finetune_weight"], by_name=True)
            logging.info("load finetune weight: %s", model_info["finetune_weight"])

    def _init_train_list(self):
        self._count = 0           # samples staged so far
        self._raw_segments = []   # (offset, length, value offset) of trajectories that still need device GAE
        # valid rows of the raw stores: up to the end of the last raw trajectory (rows of trajectories that came with their
        # advantages are gaps, so the rollout's row count can be past the stores' capacity)
        self._raw_steps.n = self._raw_values.n = 0

    # -- data path ---------------------------------------------------------------------------
    def prepare_data(self, train_data, **kwargs):
        """`ring_rows` = (env_index, first_step, n_steps) instead of `cur_state`: the trajectory's frames are the ones the
        learner-side batched predict() already uploaded (model.keep_predict_obs); they are copied device to device."""
        ro = self.actor.rollout
        ring_rows = train_data.get("ring_rows")
        n = int(ring_rows[2]) if ring_rows is not None else len(train_data["cur_state"])
        ro.n = self._count
        ro.reserve(self._count + n)
        sl = slice(self._count, self._count + n)
        if ring_rows is not None:
            ring = self.actor._obs_ring
            e, t0 = int(ring_rows[0]), int(ring_rows[1]) % ring["T"]
            if t0 + n > ring["T"]:
                raise ValueError("trajectory wraps around the observation ring")
            ro.obs[sl].copy_(ring["obs"][t0:t0 + n, e], non_blocking=True)
        else:
            stage_h2d(ro.obs[sl], np.asarray(train_data["cur_state"]), self.actor._np_dt)
        # int32 [n] actions, or float32 [n, A] for a DiagGaussian actor
        stage_h2d(ro.action[sl], train_data["action"], np.float32 if ro.action.dim() == 2 else np.int32)
        stage_h2d(ro.old_logp[sl], train_data["logp"], np.float32)
        if "adv" in train_data:
            stage_h2d(ro.adv[sl], train_data["adv"], np.float32)
            stage_h2d(ro.old_v[sl], train_data["old_value"], np.float32)
            stage_h2d(ro.target_v[sl], train_data["target_value"], np.float32)
        else:
            value = np.ascontiguousarray(train_data["value"], np.float32).reshape(-1)
            if value.size != n + 1:
                raise ValueError("raw trajectory needs value[T+1] (bootstrap appended), got %d for T=%d" % (value.size, n))
            steps, values = self._raw_steps, self._raw_values
            voff = self._count + len(self._raw_segments)          # every earlier raw trajectory holds one bootstrap value more
            steps.reserve(self._count + n)
            values.reserve(voff + n + 1)
            stage_h2d(values.val[voff:voff + n + 1], value, np.float32)     # staged (asynchronous): no host sync per trajectory
            stage_h2d(steps.rew[sl], np.asarray(train_data["reward"]).reshape(-1), np.float32)
            stage_h2d(steps.don[sl], np.asarray(train_data["done"]).reshape(-1).astype(np.bool_, copy=False).view(np.uint8), np.uint8)
            steps.n, values.n = self._count + n, voff + n + 1
            self._raw_segments.append((self._count, n, voff))
        self._count += n
        ro.n = self._count

    def _device_gae(self):
        """GAE of the raw trajectories on the device: one launch over [E, T] when they are equally long and adjacent (the
        value buffer is then exactly [E, T+1]), else one launch per trajectory."""
        ro = self.actor.rollout
        lib = self.actor.net.lib
        segs = self._raw_segments
        if not segs:
            return
        steps, values = self._raw_steps, self._raw_values
        same = len({s[1] for s in segs}) == 1 and all(segs[i][0] + segs[i][1] == segs[i + 1][0] and segs[i][2] + segs[i][1] + 1 == segs[i + 1][2]
                                                      for i in range(len(segs) - 1))
        groups = [(segs[0][0], segs[0][1], segs[0][2], len(segs))] if same else [(o, t, v, 1) for o, t, v in segs]
        for off, t, voff, count in groups:
            check(lib.xtb_gae(_ptr(values.val[voff:]), _ptr(steps.rew[off:]), _ptr(steps.don[off:]), count, t, GAMMA, LAM,
                              int(self.sign_clip_reward), _ptr(ro.adv[off:]), _ptr(ro.old_v[off:]), _ptr(ro.target_v[off:]), stream_ptr()))
        self._raw_segments = []

    def train(self, **kwargs):
        """xt/algorithm/ppo/ppo.py:64-77."""
        if self._count == 0:
            raise ValueError("need at least one array to concatenate")   # np.concatenate([]) in the reference
        self._device_gae()
        loss = self.actor.train_device(self._count)
        self._init_train_list()
        return loss

    def predict(self, state):
        """xt/algorithm/ppo/ppo.py:87-95."""
        if not isinstance(state, (list, tuple)):
            state = state.reshape((1,) + state.shape)
        else:
            state = list(map(lambda x: x.reshape((1,) + x.shape), state))
            state = np.vstack(state)
        return self.actor.predict(state)
