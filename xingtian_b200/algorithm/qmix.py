"""QMixAlg (xt/algorithm/qmix/qmix_alg.py) over QMixModel: the host episode buffer, the agents' input assembly, the
epsilon-greedy selector and the training batch preparation.  The network work is QMixModel's (xtb_qmix_train /
xtb_qmix_infer); everything here is NumPy on the host and draws from the global np.random stream in the reference's
order, so a seeded run samples the same episodes and picks the same actions.  With alg_config DEVICE_REPLAY the episode
ring lives in HBM instead (DeviceEpisodeReplay) and the batch is assembled there, inside the model's training graph."""
import ctypes as C
import logging
import os

import numpy as np
import torch

from .. import capi
from ..engine import _ptr, stream_ptr
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


class EpisodeRing(object):
    """ReplayBuffer's bookkeeping without its arrays: the ring position, the stored count and the draw of the episode ids,
    with the same rules and the same np.random calls."""

    def __init__(self, buffer_size):
        self.buffer_size = buffer_size
        self.buffer_index = self.episodes_in_buffer = 0

    def insert(self, k):
        """Advance over k new episodes as insert_episode_batch does (a batch running past the end is split there) -> the
        slot of each, in order."""
        if self.buffer_index + k <= self.buffer_size:
            slots = list(range(self.buffer_index, self.buffer_index + k))
            self.buffer_index += k
            self.episodes_in_buffer = max(self.episodes_in_buffer, self.buffer_index)
            self.buffer_index %= self.buffer_size
            return slots
        left = self.buffer_size - self.buffer_index
        return self.insert(left) + self.insert(k - left)

    def can_sample(self, batch_size):
        return self.episodes_in_buffer >= batch_size

    def sample(self, batch_size):
        """The ids ReplayBuffer.sample would gather: all of them, undrawn, when exactly batch_size are stored."""
        if not self.can_sample(batch_size):
            raise ValueError("{} episodes stored, {} requested".format(self.episodes_in_buffer, batch_size))
        if self.episodes_in_buffer == batch_size:
            return np.arange(batch_size)
        return np.random.choice(self.episodes_in_buffer, batch_size, replace=False)


# The fields of a packed episode row (xtb200.h, xtb_episode_replay): scheme key and stored dtype, in row order
ROW_FIELDS = (("state", np.float32), ("obs", np.float32), ("actions", np.int32), ("actions_onehot", np.float32),
              ("avail_actions", np.int32), ("reward", np.float32), ("terminated", np.uint8), ("filled", np.int64))


class EpisodeRowPacker(object):
    """One episode as DeviceEpisodeReplay stores it: the values ReplayBuffer's row would hold after insert_episode_batch
    (EpisodeBatch.update on a one-episode scratch batch: the scheme dtypes, the actions one-hot, a caller's
    actions_onehot written after actions winning), packed into one byte row of the device layout.  The one-hot is kept
    as float32: the host path rounds its float64 to float32 once when it stages the batch, as this does."""

    def __init__(self, scheme, groups, max_seq_length, preprocess):
        self.scratch = EpisodeBatch(scheme, groups, 1, max_seq_length, preprocess=preprocess)
        self.T, self.n, self.A = max_seq_length, groups["agents"], self.scratch.scheme["avail_actions"]["vshape"][0]
        derived = {new_key for new_key, _ in self.scratch.preprocess.values()}
        self.required = [k for k in self.scratch.data if k not in derived]
        self.shapes = [(key, self.scratch.data[key].shape[1:], dt) for key, dt in ROW_FIELDS]
        sizes = [int(np.prod(s)) * np.dtype(dt).itemsize for _, s, dt in self.shapes]
        self.offsets = [int(o) for o in np.cumsum([0] + [(s + 15) // 16 * 16 for s in sizes])]
        self.row_bytes = self.offsets[-1]

    def pack(self, data):
        """data {key: [T, ...]} -> the uint8 row.  ValueError for a missing field (the device ring keeps no earlier
        episode's values to fall back on), an action of the first T - 1 steps outside [0, n_actions) or a filled sum
        outside [0, T]: the training batch reads them as indices and lengths."""
        missing = [k for k in self.required if k not in data]
        if missing:
            raise ValueError("the device replay stores whole episodes: {} missing".format(missing))
        sb = self.scratch
        act = np.array(data["actions"], dtype=sb.scheme["actions"]["dtype"]).reshape(sb.data["actions"].shape)
        bad = (act[:, :-1] < 0) | (act[:, :-1] >= self.A)
        if np.any(bad):
            raise ValueError("actions must be in [0, {}), got {}".format(self.A, act[:, :-1][bad][0]))
        sb.update(data, mark_filled=False)
        filled = int(np.sum(sb.data["filled"]))
        if not 0 <= filled <= self.T:
            raise ValueError("filled sums to {}, not in [0, {}]".format(filled, self.T))
        row = np.zeros(self.row_bytes, np.uint8)
        for (key, shape, dt), o in zip(self.shapes, self.offsets):
            v = np.ascontiguousarray(sb.data[key][0], dtype=dt).reshape(-1).view(np.uint8)
            row[o:o + v.size] = v
        return row

    def fields(self, row):
        """{key: array} views of a packed row, in their stored dtypes and [T, ...] shapes."""
        return {key: row[o:o + int(np.prod(shape)) * np.dtype(dt).itemsize].view(dt).reshape(shape)
                for (key, shape, dt), o in zip(self.shapes, self.offsets)}


class DeviceEpisodeReplay(EpisodeRing):
    """ReplayBuffer in HBM (xtb_episode_replay): episodes are packed on the host (EpisodeRowPacker) and stored with one
    staged upload each; the ring bookkeeping and the draws stay on the host (EpisodeRing).  The training batch is
    gathered on the device from the drawn ids, by gather() or inside the models' train_replay."""

    def __init__(self, scheme, groups, buffer_size, max_seq_length, preprocess, obs_last_action, obs_agent_id, device=None):
        super().__init__(buffer_size)
        self.packer = EpisodeRowPacker(scheme, groups, max_seq_length, preprocess)
        sh = self.packer.scratch.scheme
        self.T, self.n, self.A = max_seq_length, groups["agents"], self.packer.A
        self.obs_dim, self.state_dim = int(np.prod(sh["obs"]["vshape"])), int(np.prod(sh["state"]["vshape"]))
        self.width = self.obs_dim + (self.A if obs_last_action else 0) + (self.n if obs_agent_id else 0)
        self.switches = (int(bool(obs_last_action)), int(bool(obs_agent_id)))
        self.device = device
        self._bufs = {}
        self._create()

    def _create(self):
        """The native ring (one device allocation)."""
        self.device = torch.device("cuda", torch.cuda.current_device()) if self.device is None else torch.device(self.device)
        self.handle = C.c_void_p()
        with torch.cuda.device(self.device):
            capi.check(capi.lib().xtb_episode_replay_create(self.buffer_size, self.T - 1, self.n, self.A, self.obs_dim, self.state_dim,
                                                            *self.switches, C.byref(self.handle)))
        if capi.lib().xtb_episode_replay_row_bytes(self.handle) != self.packer.row_bytes:
            raise RuntimeError("episode row layout disagrees with the library's")

    def _store(self, slot, row):
        """One packed row into ring slot `slot` (one staged upload)."""
        capi.check(capi.lib().xtb_episode_replay_add(self.handle, slot, row.ctypes.data, row.nbytes, stream_ptr()))

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                capi.lib().xtb_episode_replay_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:   # interpreter shutdown
            pass

    def insert_episode_batch(self, ep):
        """Store ep's episodes at the ring position, as ReplayBuffer.insert_episode_batch; every episode is checked and
        packed (ValueError) before anything is stored."""
        rows = [ep.data] if ep.batch_size == 1 else [ep[i:i + 1].data for i in range(ep.batch_size)]
        packed = [self.packer.pack(r) for r in rows]
        before = self.buffer_index, self.episodes_in_buffer
        try:
            for row, slot in zip(packed, self.insert(len(packed))):
                self._store(slot, row)
        except Exception:    # a refused store (a communicator installed, say) leaves the ring where it was
            self.buffer_index, self.episodes_in_buffer = before
            raise

    def buffers(self, B):
        """Device buffers of a gathered B-episode batch (xtb_episode_batch), overwritten by the next gather of that size."""
        b = self._bufs.get(B)
        if b is None:
            T, L, n, A, dev = self.T, self.T - 1, self.n, self.A, self.device
            f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
            b = dict(obs=torch.empty(B, T, n, self.width, **f32), raw_obs=torch.empty(B, T, n, self.obs_dim, **f32),
                     seq_len=torch.empty(B * n, **i32), avail=torch.empty(B, T, n, A, **f32), actions=torch.empty(B, L, n, **i32),
                     state=torch.empty(B, L, self.state_dim, **f32), next_state=torch.empty(B, L, self.state_dim, **f32),
                     reward=torch.empty(B, L, **f32), terminated=torch.empty(B, L, **f32), mask=torch.empty(B, L, **f32),
                     max_t=torch.zeros(1, **i32))
            bt = capi.EpisodeBatch()
            for k in ("obs", "raw_obs", "seq_len", "avail", "actions", "state", "next_state", "reward", "terminated", "mask"):
                setattr(bt, k, b[k].data_ptr())
            b["batch"] = bt
            self._bufs[B] = b
        return b

    def gather(self, ids):
        """The training batch of episodes `ids` (xtb_episode_replay_gather) -> {name: device tensor} of buffers()."""
        ids = np.ascontiguousarray(ids, np.int32)
        b = self.buffers(len(ids))
        capi.check(capi.lib().xtb_episode_replay_gather(self.handle, len(ids), ids.ctypes.data, C.byref(b["batch"]), _ptr(b["max_t"]),
                                                        stream_ptr()))
        return b


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


def _device_replay_flag(alg_config):
    """alg_config DEVICE_REPLAY (or device_replay), a bool, default False; checked before anything touches CUDA."""
    given = [(k, alg_config[k]) for k in ("DEVICE_REPLAY", "device_replay") if k in alg_config]
    for k, v in given:
        if not isinstance(v, (bool, np.bool_)):
            raise ValueError("{} must be a bool, got {!r}".format(k, v))
    if len(given) == 2 and bool(given[0][1]) != bool(given[1][1]):
        raise ValueError("DEVICE_REPLAY and device_replay disagree")
    return bool(given[0][1]) if given else False


@Registers.algorithm
class QMixAlg(Algorithm):
    """QMixAlg (qmix_alg.py:102-410).

    alg_config DEVICE_REPLAY True (or device_replay) keeps the episode ring in HBM (DeviceEpisodeReplay) in the train
    scene: prepare_data packs and uploads each episode once and draws the ids with the host's np.random calls, and
    train() gathers the batch and steps the model in one graph (the model's train_replay)."""

    device_replay = False

    def __init__(self, model_info, alg_config, **kwargs):
        device_replay = _device_replay_flag(alg_config)
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
        # the model's acting assembles the inputs as build_inputs does
        model_info["actor"]["model_config"]["obs_last_action"] = bool(alg_config["obs_last_action"])
        model_info["actor"]["model_config"]["obs_agent_id"] = bool(alg_config["obs_agent_id"])
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
        # the device ring serves the learner only: the explore scene allocates nothing on the device
        self.device_replay = device_replay and model_info["actor"]["scene"] == "train"
        if self.device_replay:
            self.buffer = DeviceEpisodeReplay(self.scheme, self.groups, alg_config["buffer_size"], env_info["episode_limit"] + 1,
                                              self.preprocess, alg_config["obs_last_action"], alg_config["obs_agent_id"],
                                              device=getattr(self.actor, "device", None))
        else:
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

    def predict_with_selector_envs(self, obs, avail, reset, t_env, test_mode, uniforms=None):
        """predict_with_selector for N environments in one device call (the model's act, environment e in slot e) ->
        int32 actions [N, n_agents].  obs [N, n_agents, obs_shape] and avail [N, n_agents, n_actions] are the step's
        observations and available actions; reset [N] marks the environments whose episode starts at this step (the
        t_ep == 0 of build_inputs and reset_hidden_state).  Epsilon follows the selector's schedule per environment (t_env
        a scalar or [N]), 0 in test mode; selector.epsilon is left as the host selector would leave it after the last
        environment.  uniforms: [N, 2, n_agents] float64 (selector_uniforms draws the host selector's numbers), or None
        for Philox draws on the device."""
        N = np.shape(obs)[0]
        t = np.broadcast_to(np.asarray(t_env), (N,))
        eps = np.zeros(N) if test_mode else np.array([self.selector.schedule.eval(x) for x in t], np.float64)
        self.selector.epsilon = 0.0 if test_mode else self.selector.schedule.eval(t[-1])
        return self.actor.act(obs, avail, reset, eps, uniforms)

    @staticmethod
    def selector_uniforms(N, n_agents):
        """The uniforms EpsilonGreedyActionSelector.select_action draws from the global np.random stream, one
        environment after another -> float64 [N, 2, n_agents]: per environment n_agents rand values (the epsilon tests),
        then one per agent row for np.random.choice (which draws one random_sample and inverts the CDF)."""
        out = np.empty((N, 2, n_agents), np.float64)
        for e in range(N):
            out[e, 0] = np.random.rand(1, n_agents)[0]
            out[e, 1] = [np.random.random_sample() for _ in range(n_agents)]
        return out

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
        (episode_num - last sync) / target_update_interval >= 1.  With the device replay the batch is the drawn ids and
        the step is the model's train_replay: one upload of the ids, one graph, one download of the loss and max_t."""
        if self.train_batch is None:
            return np.nan
        episode_num = kwargs.get("episode_num")
        if not episode_num:
            raise KeyError("need episode num to update target network")
        if self.device_replay:
            self.train_times += 1
            loss, max_ep_t = self.actor.train_replay(self.buffer, self.train_batch)
            self._after_train(episode_num, max_ep_t)
            return loss
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
        self._after_train(episode_num, max_ep_t)
        return loss

    def _after_train(self, episode_num, max_ep_t):
        """The explore-agent sync after every step, the target sync once per target_update_interval episodes."""
        self.actor.assign_explore_agent()
        if (episode_num - self.last_target_update_episode) / self.alg_config["target_update_interval"] >= 1.0:
            self.actor.assign_targets()
            logging.info("episode-%s, target Q network params replaced (train %d, seq-len %d)", episode_num, self.train_times,
                         max_ep_t)
            self.last_target_update_episode = episode_num

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
