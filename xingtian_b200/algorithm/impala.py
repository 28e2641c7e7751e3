"""IMPALA algorithm (xt/algorithm/impala/impala.py:31-189): the learner-side V-trace variant and one Keras fit per
BATCH_SIZE slice, trained with ImpalaMlp / ImpalaCnn."""
import os

import numpy as np
import torch

from ..capi import ImpalaTraj, check
from ..engine import _ptr, stage_h2d, stream_ptr
from ..model.impala_keras import FIT_BATCH
from ..registry import Registers, import_config
from .base import Algorithm, FIFODistPolicy

# xt/algorithm/impala/default_config.py
GAMMA = 0.99
BATCH_SIZE = 512


def slice_orders(n_train, batch_size):
    """The np.random call sequence of IMPALA.train (impala.py:62-84): one Keras fit, hence one
    np.random.shuffle(np.arange(len)), per consecutive BATCH_SIZE slice, in order.  Returns the training rows, slice by
    slice, in the order the minibatches read them."""
    parts = []
    for s0 in range(0, n_train, batch_size):
        idx = np.arange(min(batch_size, n_train - s0))
        np.random.shuffle(idx)
        parts.append(idx + s0)
    return np.concatenate(parts)


@Registers.algorithm
class IMPALA(Algorithm):
    """Buffers whole trajectories (L+1 states, L steps) on the device and trains them in one native call: forward of
    every state, V-trace, then a Keras fit epoch per BATCH_SIZE slice -- replayed as a CUDA graph."""

    def __init__(self, model_info, alg_config, **kwargs):
        import_config(globals(), alg_config)
        super().__init__(alg_name="impala", model_info=model_info["actor"], alg_config=alg_config)
        self.async_flag = False
        self.episode_len = int(alg_config.get("episode_len", 128))
        self.dist_model_policy = FIFODistPolicy(alg_config["instance_num"], prepare_times=self._prepare_times_per_train)
        self._store, self._n_traj = None, 0
        self.pg_adv = self.target_value = None    # device views of the last train call's V-trace outputs

    def _reserve(self, n_traj):
        """Grow-only device trajectory store (addresses stay put between calls, so the captured train graph is replayed)."""
        st = self._store
        if st is not None and st["cap"] >= n_traj:
            return st
        cap = max(n_traj, 2 * (st["cap"] if st else 0))
        L, A, dev = self.episode_len, self.actor.action_dim, self.actor.device
        new = dict(cap=cap,
                   obs=torch.empty((cap * (L + 1),) + tuple(self.actor.state_dim), dtype=self.actor._obs_dt, device=dev),
                   behav=torch.empty(cap * L, A, dtype=torch.float32, device=dev),
                   amat=torch.empty(cap * L, A, dtype=torch.float32, device=dev),
                   reward=torch.empty(cap * L, dtype=torch.float32, device=dev),
                   done=torch.empty(cap * L, dtype=torch.uint8, device=dev),
                   order=torch.empty(cap * L, dtype=torch.int32, device=dev),
                   obs_idx=torch.empty(cap * L, dtype=torch.int32, device=dev),
                   pg_adv=torch.empty(cap * L, dtype=torch.float32, device=dev),
                   tv=torch.empty(cap * L, dtype=torch.float32, device=dev),
                   loss=torch.zeros(cap * L, dtype=torch.float32, device=dev))
        if st is not None and self._n_traj:
            for k, per in (("obs", L + 1), ("behav", L), ("amat", L), ("reward", L), ("done", L)):
                new[k][:self._n_traj * per].copy_(st[k][:self._n_traj * per])
        self._store = new
        return new

    def _data_proc(self, episode_data):
        """impala.py:108-118, checked against episode_len: states [L+1, ...] (the last the bootstrap state), real_action
        one-hot [L, A], action (behaviour probabilities) [L, A], reward [L], done [L]."""
        L, A = self.episode_len, self.actor.action_dim
        states = np.asarray(episode_data["cur_state"])
        actions = np.asarray(episode_data["real_action"], np.float32)
        pred_a = np.asarray(episode_data["action"], np.float32)
        rewards = np.asarray(episode_data["reward"], np.float32).reshape(-1)
        dones = np.asarray(episode_data["done"]).reshape(-1)
        shapes = (states.shape[:1], actions.shape, pred_a.shape, rewards.shape, dones.shape)
        if shapes != ((L + 1,), (L, A), (L, A), (L,), (L,)):
            raise ValueError("IMPALA: a trajectory of episode_len %d with %d actions needs cur_state [%d, ...], real_action, "
                             "action [%d, %d], reward, done [%d]; got %s" % (L, A, L + 1, L, A, L, shapes))
        return states, actions, dones.astype(np.bool_), pred_a, rewards

    def prepare_data(self, train_data, **kwargs):
        """impala.py:96-105 -- staged straight into the device store (pinned ring, asynchronous)."""
        states, actions, dones, pred_a, rewards = self._data_proc(train_data)
        L, k = self.episode_len, self._n_traj
        st = self._reserve(k + 1)
        stage_h2d(st["obs"][k * (L + 1):(k + 1) * (L + 1)], states, self.actor._np_dt)
        stage_h2d(st["amat"][k * L:(k + 1) * L], actions, np.float32)
        stage_h2d(st["behav"][k * L:(k + 1) * L], pred_a, np.float32)
        stage_h2d(st["reward"][k * L:(k + 1) * L], rewards, np.float32)
        stage_h2d(st["done"][k * L:(k + 1) * L], dones.view(np.uint8), np.uint8)
        self._n_traj = k + 1

    def train(self, **kwargs):
        """impala.py:62-84: V-trace over the stored trajectories, one actor.train (Keras fit) per BATCH_SIZE slice, mean
        of the slice losses."""
        if self._n_traj == 0:
            raise ValueError("need at least one array to concatenate")
        n, L, st, model = self._n_traj, self.episode_len, self._store, self.actor
        n_train = n * L
        count = (n_train + BATCH_SIZE - 1) // BATCH_SIZE
        stage_h2d(st["order"][:n_train], slice_orders(n_train, BATCH_SIZE), np.int32)
        net = model.net
        net.ensure_batch(n * (L + 1))
        tr = ImpalaTraj(_ptr(st["obs"]), _ptr(st["behav"]), _ptr(st["amat"]), _ptr(st["reward"]), _ptr(st["done"]))
        check(net.lib.xtb_impala_keras_train(net.handle, model.opt.handle, tr, n, L, int(BATCH_SIZE), FIT_BATCH, _ptr(st["order"]),
                                             _ptr(st["obs_idx"]), float(GAMMA), float(model.ent_coef), net.tid[model.logit_name],
                                             net.tid[model.value_name], _ptr(st["pg_adv"]), _ptr(st["tv"]), _ptr(st["loss"]),
                                             1 if model.use_graph else 0, stream_ptr()))
        self.pg_adv, self.target_value = st["pg_adv"][:n_train], st["tv"][:n_train]
        self._n_traj = 0
        return float(st["loss"][:count].double().mean().cpu())

    def save(self, model_path, model_index):
        """impala.py:86-93."""
        actor_name = "actor" + str(model_index).zfill(5)
        actor_name = self.actor.save_model(os.path.join(model_path, actor_name))
        return [actor_name.split("/")[-1]]

    def predict(self, state):
        """impala.py:107-113: [probs [1, A], value [1, 1]] of one state."""
        state = state.reshape((1,) + state.shape)
        return self.actor.predict([state, np.zeros((1, 1))])
