"""QMixAlg (xt/algorithm/qmix/qmix_alg.py) over QMixModel: the host episode buffer, the agents' input assembly, the
epsilon-greedy selector and the training batch preparation.  The network work is QMixModel's (xtb_qmix_train /
xtb_qmix_infer); everything here is NumPy on the host and draws from the global np.random stream in the reference's
order, so a seeded run samples the same episodes and picks the same actions."""
import logging
import os

import numpy as np

from ..registry import Registers
from .base import Algorithm, ZFILL_LENGTH


class EpisodeBatch(object):
    """The episode store of the reference's EpisodeBatchNP (xt/algorithm/qmix/episode_buffer_np.py, after pymarl): every
    field is [batch, max_seq_length, (group members,) *vshape] of its scheme dtype (float32 when none is given), plus the
    reserved int64 `filled` flag.  A preprocess {key: (new_key, [transforms])} derives `new_key` from `key` on every
    update; its shape and dtype come from the transforms (OneHot gives float64, as np.float)."""

    def __init__(self, scheme, groups, batch_size, max_seq_length, data=None, preprocess=None):
        self.scheme, self.groups = dict(scheme), groups
        self.batch_size, self.max_seq_length = batch_size, max_seq_length
        self.preprocess = preprocess or {}
        if data is not None:
            self.data = data
            return
        for key, (new_key, transforms) in self.preprocess.items():
            vshape, dtype = self.scheme[key]["vshape"], self.scheme[key]["dtype"]
            for tr in transforms:
                vshape, dtype = tr.infer_output_info(vshape, dtype)
            self.scheme[new_key] = dict(vshape=vshape, dtype=dtype)
            if "group" in self.scheme[key]:
                self.scheme[new_key]["group"] = self.scheme[key]["group"]
        if "filled" in self.scheme:
            raise KeyError('"filled" is a reserved key for masking')
        self.scheme["filled"] = dict(vshape=(1,), dtype=np.int64)
        self.data = {}
        for key, info in self.scheme.items():
            vshape = info["vshape"]
            vshape = (vshape,) if isinstance(vshape, int) else tuple(vshape)
            members = (groups[info["group"]],) if info.get("group") else ()
            self.data[key] = np.zeros((batch_size, max_seq_length) + members + vshape, dtype=info.get("dtype", np.float32))

    @staticmethod
    def _slices(bs, ts):
        return tuple(slice(i, i + 1) if isinstance(i, int) else i for i in (bs, ts))

    def update(self, data, bs=slice(None), ts=slice(None), mark_filled=True):
        """Write `data` {key: array} into rows bs, steps ts (each value reshaped to the target's shape); the first key
        also sets `filled` there unless mark_filled is False."""
        sl = self._slices(bs, ts)
        for key, val in data.items():
            if key not in self.data:
                raise KeyError("{} not found in transition or episode data".format(key))
            if mark_filled:
                self.data["filled"][sl] = 1
                mark_filled = False
            dest = self.data[key][sl]
            dest[...] = np.array(val, dtype=self.scheme[key].get("dtype", np.float32)).reshape(dest.shape)
            if key in self.preprocess:
                new_key, transforms = self.preprocess[key]
                v = dest
                for tr in transforms:
                    v = tr.transform(v)
                self.data[new_key][sl] = v

    def __getitem__(self, item):
        if isinstance(item, str):
            return self.data[item]
        idx = item if isinstance(item, (slice, list, np.ndarray)) else slice(item, item + 1)
        sub = {k: v[idx] for k, v in self.data.items()}
        n = len(range(*idx.indices(self.batch_size))) if isinstance(idx, slice) else len(idx)
        return EpisodeBatch(self.scheme, self.groups, n, self.max_seq_length, data=sub)

    def max_t_filled(self):
        """The most filled steps of any episode."""
        return np.sum(self.data["filled"], 1).max(0)[0]


class ReplayBuffer(EpisodeBatch):
    """ReplayBufferNP: a ring of buffer_size episodes, sampled uniformly without replacement."""

    def __init__(self, scheme, groups, buffer_size, max_seq_length, preprocess=None):
        super().__init__(scheme, groups, buffer_size, max_seq_length, preprocess=preprocess)
        self.buffer_size = buffer_size
        self.buffer_index = self.episodes_in_buffer = 0

    def insert_episode_batch(self, ep):
        """Store ep's episodes at the ring position (its arrays are reshaped to [episodes, steps, ...]); a batch that
        would run past the end is split there."""
        if self.buffer_index + ep.batch_size <= self.buffer_size:
            rows = slice(self.buffer_index, self.buffer_index + ep.batch_size)
            self.update(ep.data, rows, slice(0, ep.max_seq_length), mark_filled=False)
            self.buffer_index += ep.batch_size
            self.episodes_in_buffer = max(self.episodes_in_buffer, self.buffer_index)
            self.buffer_index %= self.buffer_size
        else:
            left = self.buffer_size - self.buffer_index
            self.insert_episode_batch(ep[0:left])
            self.insert_episode_batch(ep[left:])

    def can_sample(self, batch_size):
        return self.episodes_in_buffer >= batch_size

    def sample(self, batch_size):
        if not self.can_sample(batch_size):
            raise ValueError("{} episodes stored, {} requested".format(self.episodes_in_buffer, batch_size))
        if self.episodes_in_buffer == batch_size:
            return self[:batch_size]
        return self[np.random.choice(self.episodes_in_buffer, batch_size, replace=False)]


class OneHot(object):
    """OneHotNp: integer [..., 1] -> float64 one-hot [..., out_dim]."""

    def __init__(self, out_dim, dtype=np.float64):
        self.out_dim, self.dtype = out_dim, dtype

    def transform(self, x):
        x = np.asarray(x)
        return np.eye(self.out_dim)[x.reshape(-1)].reshape(x.shape[:-1] + (self.out_dim,)).astype(self.dtype)

    def infer_output_info(self, vshape, dtype):
        return (self.out_dim,), self.dtype


class DecayThenFlatSchedule(object):
    """pymarl's schedule: "linear" max(finish, start - t (start - finish) / time_length), or "exp"."""

    def __init__(self, start, finish, time_length, decay="exp"):
        self.start, self.finish, self.time_length, self.decay = start, finish, time_length, decay
        self.delta = (start - finish) / time_length
        if decay == "exp":
            self.exp_scaling = -time_length / np.log(finish) if finish > 0 else 1

    def eval(self, t):
        if self.decay == "linear":
            return max(self.finish, self.start - self.delta * t)
        if self.decay == "exp":
            return min(self.start, max(self.finish, np.exp(-t / self.exp_scaling)))
        raise KeyError("invalid decay-{} configured".format(self.decay))


class EpsilonGreedyActionSelector(object):
    """Greedy over the available actions, or with probability epsilon a uniform draw among them.  Per call: one
    np.random.rand of [batch, agents], then one np.random.choice per agent row."""

    def __init__(self, args):
        self.schedule = DecayThenFlatSchedule(args["epsilon_start"], args["epsilon_finish"], args["epsilon_anneal_time"],
                                              decay="linear")
        self.epsilon = self.schedule.eval(0)

    def select_action(self, agent_inputs, avail_actions, t_env, test_mode=False):
        self.epsilon = 0.0 if test_mode else self.schedule.eval(t_env)
        masked = agent_inputs.copy()
        masked[avail_actions < 1e-6] = -float("inf")
        pick_random = (np.random.rand(*agent_inputs[:, :, 0].shape) < self.epsilon).astype(np.int64)
        n_agents, n_act = avail_actions.shape[1], avail_actions.shape[2]
        probs = (avail_actions / np.expand_dims(avail_actions.sum(-1), -1)).astype(np.float64).reshape(-1, n_act)
        random_actions = np.array([np.random.choice(n_act, p=p) for p in probs]).reshape((-1, n_agents))
        return pick_random * random_actions + (1 - pick_random) * masked.argmax(axis=2)


@Registers.algorithm
class QMixAlg(Algorithm):
    """QMixAlg (qmix_alg.py:102-410)."""

    def __init__(self, model_info, alg_config, **kwargs):
        env_info = alg_config["env_attr"]
        alg_config.update({"n_agents": env_info["n_agents"], "n_actions": env_info["n_actions"],
                           "state_shape": env_info["state_shape"]})
        self.n_agents = alg_config["n_agents"]
        self.scheme = {
            "state": {"vshape": env_info["state_shape"]},
            "obs": {"vshape": env_info["obs_shape"], "group": "agents"},
            "actions": {"vshape": (1,), "group": "agents", "dtype": np.int64},
            "avail_actions": {"vshape": (env_info["n_actions"],), "group": "agents", "dtype": np.int32},
            "reward": {"vshape": (1,)},
            "terminated": {"vshape": (1,), "dtype": np.uint8},
            "actions_onehot": {"vshape": (env_info["n_actions"],), "dtype": np.float32, "group": "agents"},
        }
        self.obs_shape = self._get_input_shape(alg_config, self.scheme)
        model_info["actor"]["model_config"]["obs_shape"] = self.obs_shape
        model_info["actor"].update({"scene": kwargs.get("scene", "train")})
        super().__init__(alg_name="QMixAlg", model_info=model_info["actor"], alg_config=alg_config)
        self.async_flag = False
        self.avail_action_num = env_info["n_actions"]
        self.fix_seq_length = env_info["episode_limit"]
        self.schedule = DecayThenFlatSchedule(alg_config["epsilon_start"], alg_config["epsilon_finish"],
                                              alg_config["epsilon_anneal_time"], decay="linear")
        self.epsilon = self.schedule.eval(0)
        self.selector = EpsilonGreedyActionSelector(alg_config)
        self.last_target_update_episode = -9999.0
        self.groups = {"agents": env_info["n_agents"]}
        self.preprocess = {"actions": ("actions_onehot", [OneHot(out_dim=alg_config["n_actions"])])}
        self.buffer = ReplayBuffer(self.scheme, self.groups, alg_config["buffer_size"], env_info["episode_limit"] + 1,
                                   preprocess=self.preprocess)
        self.train_batch = None
        self.train_times = 0

    @staticmethod
    def _get_input_shape(alg_config, scheme):
        """obs_shape plus n_actions with obs_last_action, plus n_agents with obs_agent_id."""
        shape = scheme["obs"]["vshape"]
        if alg_config["obs_last_action"]:
            shape += scheme["actions_onehot"]["vshape"][0]
        if alg_config["obs_agent_id"]:
            shape += alg_config["n_agents"]
        return shape

    def reset_hidden_state(self):
        self.actor.reset_hidden_state()

    def build_inputs(self, batch, t):
        """The agents' inputs at step t: [batch, 1, n_agents, obs (+ last action one-hot) (+ agent id one-hot)]."""
        parts = [batch["obs"][:, t]]
        if self.alg_config["obs_last_action"]:
            parts.append(np.zeros_like(batch["actions_onehot"][:, t]) if t == 0 else batch["actions_onehot"][:, t - 1])
        if self.alg_config["obs_agent_id"]:
            parts.append(np.tile(np.eye(self.n_agents)[None], (batch.batch_size, 1, 1)))
        return np.expand_dims(np.concatenate(parts, axis=-1), axis=1)

    def predict_with_selector(self, ep_batch, t_ep, t_env, test_mode):
        avail_actions = ep_batch["avail_actions"][:, t_ep]
        out_val = self.actor.infer_actions(self.build_inputs(ep_batch, t_ep))
        return self.selector.select_action(out_val, avail_actions, t_env, test_mode=test_mode)

    def save(self, model_path, model_index):
        """The explore agent's weights under model_path/actor<index>."""
        model_name = os.path.join(model_path, "actor{}".format(str(model_index).zfill(ZFILL_LENGTH)))
        self.actor.save_explore_agent_weights(model_name)
        return [model_name]

    def restore(self, model_name=None, model_weights=None):
        if model_weights is not None:
            self.actor.set_weights(model_weights)
        else:
            self.actor.restore_explorer_variable(model_name)

    def prepare_data(self, train_data, **kwargs):
        """Store one episode {key: [episode_limit + 1, ...]} and draw the next training batch once enough are stored."""
        episode = EpisodeBatch(self.scheme, self.groups, 1, self.fix_seq_length + 1, data=dict(train_data))
        self.buffer.insert_episode_batch(episode)
        bs = self.alg_config["batch_size"]
        self.train_batch = self.buffer.sample(bs) if self.buffer.can_sample(bs) else None

    def train(self, **kwargs):
        """One QMixModel.train on the drawn batch (nan without one), the explore-agent sync, and the target sync once
        (episode_num - last sync) / target_update_interval >= 1."""
        if not self.train_batch:
            return np.nan
        episode_num = kwargs.get("episode_num")
        if not episode_num:
            raise KeyError("need episode num to update target network")
        batch = self.train_batch
        max_ep_t = batch.max_t_filled()
        rewards = batch["reward"][:, :-1]
        actions = batch["actions"][:, :-1]
        terminated = batch["terminated"][:, :-1].astype(np.float32)
        mask = batch["filled"][:, :-1].astype(np.float32)
        mask[:, 1:] = mask[:, 1:] * (1 - terminated[:, :-1])
        trajectories = np.concatenate([self.build_inputs(batch, t) for t in range(batch.max_seq_length)], axis=1)
        self.train_times += 1
        loss = self.actor.train(trajectories, [max_ep_t for _ in range(batch.batch_size * self.n_agents)], batch["avail_actions"],
                                actions, batch["state"][:, :-1], batch["state"][:, 1:], rewards, terminated, mask)
        self.actor.assign_explore_agent()
        if (episode_num - self.last_target_update_episode) / self.alg_config["target_update_interval"] >= 1.0:
            self.actor.assign_targets()
            logging.info("episode-%s, target Q network params replaced (train %d, seq-len %d)", episode_num, self.train_times,
                         max_ep_t)
            self.last_target_update_episode = episode_num
        return loss

    def train_ready(self, elapsed_episode, **kwargs):
        """Ready once a batch can be sampled; before that the caller's dist_dummy_model is called (KeyError without one)."""
        if not self.buffer.can_sample(self.alg_config["batch_size"]):
            self._train_ready = False
            if not kwargs.get("dist_dummy_model"):
                raise KeyError("qmix need to dist dummy model.")
            kwargs["dist_dummy_model"]()
        else:
            self._train_ready = True
        return self._train_ready
