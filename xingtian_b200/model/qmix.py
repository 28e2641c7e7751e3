"""QMixModel on the CUDA engine (xt/model/qmix/qmix_tf.py).

The reference builds five TF sub-graphs: the explore agent (one step, hidden state carried between calls), the eval and
target agents over whole episodes, and the eval and target mixers.  Here a weight set is one flat buffer
[fc1 | GRU | fc2 | mixer] in the TF variable order of the eval_agent and eval_mixer scopes: the eval set is the one the
engine nets (fc1, fc2 and the hypernetworks) are bound to and the optimiser steps, the target set and the explore agent
are buffers of the same layout.  The training step (xtb_qmix_train), the one-step inference (xtb_qmix_infer) and the
acting of up to act_envs environments per call (xtb_qmix_act) run in libxtb200."""
import ctypes as C
import math
import os
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, Net, _ptr, stage_h2d, stream_ptr
from ..registry import Registers
from .base import XTModel

AGENT_SCOPES = ("explore_agent", "eval_agent", "target_agent")
_ALIGN = 64   # every slice of a weight set starts 256-byte aligned (the tensor-core weight refresh reads 16-byte pieces)


def _align(x):
    return (x + _ALIGN - 1) // _ALIGN * _ALIGN


@Registers.model
class QMixModel(XTModel):
    """QMixModel (qmix_tf.py:23-589).  model_info["scene"] = "explore" builds the acting network only, "train" all five.

    SCCModel shares the agent: its config fields, nets and variable table, its weight sets, the explore step and the
    native object's lifetime (the entry points named by _native)."""

    _native = "xtb_qmix"   # the native object's entry points: <_native>_infer, <_native>_act and <_native>_destroy

    def __init__(self, model_info):
        model_config = self._agent_config(model_info)
        self.lr = model_config.get("lr", 0.0005)
        self.grad_norm_clip = model_config.get("grad_norm_clip", 10)
        self.embed_dim = int(model_config["mixing_embed_dim"])
        self.use_double_q = bool(model_config.get("use_double_q", True))
        # read by the train graph only (_build_mix_net2), as in the reference
        self.hypernet_embed = int(model_config["hypernet_embed"]) if self.g_type == "train" else int(model_config.get("hypernet_embed", 1))
        super().__init__(model_info)

    def _agent_config(self, model_info):
        """The model_config fields of the agent and its training batch -> model_config."""
        model_config = model_info.get("model_config", None) or {}
        self.model_config = model_config
        self.gamma = model_config.get("gamma", 0.99)
        self.n_agents = int(model_config["n_agents"])
        self.obs_shape = int(model_config["obs_shape"])
        self.rnn_hidden_dim = int(model_config["rnn_hidden_dim"])
        self.fix_seq_length = int(model_config["episode_limit"])
        self.n_actions = int(model_config["n_actions"])
        self.batch_size = int(model_config["batch_size"])
        self.avail_action_num = self.n_actions
        self.state_dim = int(np.prod(model_config["state_shape"]))
        self.g_type = model_info.get("scene", "explore")
        # acting (act): environment slots, and which one-hots build_inputs appends to the observation
        self.act_envs = int(model_config.get("act_envs", 1))
        if self.act_envs < 1:
            raise ValueError("act_envs must be >= 1, got {}".format(self.act_envs))
        self.obs_last_action = bool(model_config.get("obs_last_action", False))
        self.obs_agent_id = bool(model_config.get("obs_agent_id", False))
        return model_config

    # ---- construction ---------------------------------------------------------------------------------------------
    def create_model(self, model_info):
        n, E, he = self.n_agents, self.embed_dim, self.hypernet_embed
        train = self.g_type == "train"
        B, L = self._agent_nets(train)
        hyp_a = dict(input_dtype="float32", state_dim=(self.state_dim,), scale=1.0, layers=[
            ("hyper_w1/dense", "dense", "obs", dict(n=he, act="relu")),
            ("hyper_w1/dense_1", "dense", "hyper_w1/dense", dict(n=E * n, act=None)),
            ("hyper_b1/dense", "dense", "obs", dict(n=E, act=None)),
            ("hyper_w_final/dense", "dense", "obs", dict(n=he, act="relu")),
            ("hyper_w_final/dense_1", "dense", "hyper_w_final/dense", dict(n=E, act=None)),
            ("val_for_bias/dense", "dense", "obs", dict(n=E, act="relu")),
            ("val_for_bias/dense_1", "dense", "val_for_bias/dense", dict(n=1, act=None)),
        ])
        self.hyper = Net(hyp_a, max_batch=B * L, device=self.device)
        o_hyp = _align(self.agent_size)
        self.n_params = o_hyp + self.hyper.n_params
        for name, (o, shape) in self.hyper.ptable.items():
            self.mixer_vars[name] = (o_hyp + o, shape)
        self._weight_sets([(self.hyper, o_hyp)], target_agent=True)
        dev = self.device
        self.opt = None
        if train:
            starts = [o for o, _ in list(self.agent_vars.values()) + list(self.mixer_vars.values())] + [self.n_params]
            flat = SimpleNamespace(params=self.params, n_params=self.n_params, device=dev, segment_offsets=lambda: starts)
            # tf.train.RMSPropOptimizer(lr, decay=0.95, epsilon=1.5e-7, centered=True) with clip_by_norm of every gradient
            self.opt = Adam(flat, self.lr, clip_mode=capi.CLIP_PER_TENSOR, clip=float(self.grad_norm_clip))
            self.opt.use_rmsprop(decay=0.95, epsilon=1.5e-7)
        desc = capi.QmixDesc()
        desc.batch, desc.episode_limit, desc.n_agents = B, L, n
        desc.use_double_q, desc.gamma, desc.gru_off = int(self.use_double_q), float(self.gamma), self.gru_off
        desc.act_envs = self.act_envs
        self.handle = C.c_void_p()
        with torch.cuda.device(dev):
            check(capi.lib().xtb_qmix_create(self.fc1.handle, self.fc2.handle, self.hyper.handle, C.byref(desc), C.byref(self.handle)))
        self._acting_state()
        return self.fc1

    def _agent_nets(self, train):
        """fc1 and fc2 for the scene's training batch and the agent's variable table -> (batch, episode limit).  The
        explore scene keeps a minimal training shape: only the one-step inference and acting run.  Both nets also hold
        the act_envs n_agents rows of acting."""
        H, A, n = self.rnn_hidden_dim, self.n_actions, self.n_agents
        B, L = (self.batch_size, self.fix_seq_length) if train else (1, 1)
        fc1_a = dict(input_dtype="float32", state_dim=(self.obs_shape,), scale=1.0,
                     layers=[("dense", "dense", "obs", dict(n=H, act="relu"))])
        fc2_a = dict(input_dtype="float32", state_dim=(H,), scale=1.0, layers=[("dense_1", "dense", "obs", dict(n=A, act=None))])
        rows = max(B * (L + 1) * n, self.act_envs * n)
        self.fc1 = Net(fc1_a, max_batch=rows, device=self.device)
        self.fc2 = Net(fc2_a, max_batch=rows, device=self.device)
        gru = OrderedDict([("rnn/gru_cell/gates/kernel", (2 * H, 2 * H)), ("rnn/gru_cell/gates/bias", (2 * H,)),
                           ("rnn/gru_cell/candidate/kernel", (2 * H, H)), ("rnn/gru_cell/candidate/bias", (H,))])
        self.gru_off = _align(self.fc1.n_params)
        self.o_fc2 = _align(self.gru_off + sum(int(np.prod(s)) for s in gru.values()))
        self.agent_size = self.o_fc2 + self.fc2.n_params
        # variable tables: name -> (offset in a weight set, shape), in TF variable order
        self.agent_vars, self.mixer_vars = OrderedDict(), OrderedDict()
        for name, (off, shape) in self.fc1.ptable.items():
            self.agent_vars[name] = (off, shape)
        off = self.gru_off
        for name, shape in gru.items():
            self.agent_vars[name] = (off, shape)
            off += int(np.prod(shape))
        for name, (o, shape) in self.fc2.ptable.items():
            self.agent_vars[name] = (self.o_fc2 + o, shape)
        self._B, self._L = B, L
        return B, L

    def _weight_sets(self, mixer_nets, target_agent):
        """The eval set (with its gradients), the target set and the explore agent, with fc1, fc2 and mixer_nets
        [(net, offset)] bound to the eval set.  Each sub-graph is initialised on its own, in the order the reference
        builds them; target_agent: the train graph has a target agent."""
        dev = self.device
        self.params = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.target = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.explore = torch.zeros(self.agent_size, dtype=torch.float32, device=dev)
        nets = [(self.fc1, 0), (self.fc2, self.o_fc2)] + mixer_nets
        for net, o in nets:
            net.bind_to(self.params[o:o + net.n_params], self.grads[o:o + net.n_params])
        self._init_set(self.explore, self.agent_vars)
        if self.g_type == "train":
            self._init_set(self.params, self.agent_vars)
            if target_agent:
                self._init_set(self.target, self.agent_vars)
            self._init_set(self.params, self.mixer_vars)
            self._init_set(self.target, self.mixer_vars)
        for net, _ in nets:
            net.params_changed()

    def _acting_state(self):
        """The hidden state and the one-step inference's staging, the act_envs environment slots of act (hidden state,
        last action, Philox step counter) and its staging; the training buffers are made at first use."""
        n, dev = self.n_agents, self.device
        self.hidden = torch.zeros(n, self.rnn_hidden_dim, dtype=torch.float32, device=dev)
        self._io = dict(obs1=torch.empty(n, self.obs_shape, dtype=torch.float32, device=dev),
                        q1=torch.empty(n, self.n_actions, dtype=torch.float32, device=dev))
        N, A, i32 = self.act_envs, self.n_actions, dict(dtype=torch.int32, device=dev)
        self.act_hidden = torch.zeros(N, n, self.rnn_hidden_dim, dtype=torch.float32, device=dev)
        self.act_last = torch.full((N, n), -1, **i32)
        self.act_counter = torch.zeros(N, dtype=torch.int64, device=dev)   # uint64 on the device
        self._act_seed = None
        self._act_io = dict(obs=torch.empty(N, n, self.act_obs_dim, dtype=torch.float32, device=dev), avail=torch.empty(N, n, A, **i32),
                            reset=torch.empty(N, **i32), epsilon=torch.empty(N, dtype=torch.float64, device=dev),
                            uniforms=torch.empty(N, 2, n, dtype=torch.float64, device=dev), actions=torch.empty(N, n, **i32))
        self._bufs = None
        self.net = self.fc1

    @property
    def act_obs_dim(self):
        """The raw observation width act takes: obs_shape less the one-hots build_inputs appends."""
        return self.obs_shape - (self.n_actions if self.obs_last_action else 0) - (self.n_agents if self.obs_agent_id else 0)

    def _init_set(self, flat, table):
        """TF 1.15 initialisers: glorot_uniform kernels (dense and GRUCell alike), zero biases except the GRU gates bias,
        which starts at 1.0."""
        host = flat.detach().cpu().numpy().copy()
        for name, (off, shape) in table.items():
            size = int(np.prod(shape))
            if name.endswith("kernel"):
                lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                host[off:off + size] = self._init_rng.uniform(-lim, lim, size=size).astype(np.float32)
            else:
                host[off:off + size] = 1.0 if name == "rnn/gru_cell/gates/bias" else 0.0
        flat.copy_(torch.from_numpy(host))

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                getattr(capi.lib(), self._native + "_destroy")(self.handle)
                self.handle = C.c_void_p()
        except Exception:
            pass

    # ---- weights ----------------------------------------------------------------------------------------------------
    def variables(self, flat, mixer=True):
        """{variable name (without scope): ndarray} of a weight set (self.params = eval, self.target, self.explore)."""
        host = flat.detach().cpu().numpy()
        table = list(self.agent_vars.items()) + (list(self.mixer_vars.items()) if mixer else [])
        return OrderedDict((name, host[o:o + int(np.prod(s))].reshape(s).copy()) for name, (o, s) in table)

    def get_weights(self):
        """TFVariables.get_weights of the explore agent: {"explore_agent/<variable>": ndarray} in variable order."""
        return OrderedDict(("explore_agent/" + k, v) for k, v in self.variables(self.explore, mixer=False).items())

    def set_weights(self, weights):
        """TFVariables.set_weights: assigns the explore-agent variables named in `weights`; KeyError when none is."""
        host = self.explore.detach().cpu().numpy().copy()
        hit = 0
        for key, value in weights.items():
            name = key[len("explore_agent/"):] if key.startswith("explore_agent/") else None
            if name not in self.agent_vars:
                continue
            off, shape = self.agent_vars[name]
            v = np.asarray(value, dtype=np.float32)
            if tuple(v.shape) != tuple(shape):
                raise ValueError("weight {}: shape {} != {}".format(key, v.shape, shape))
            host[off:off + v.size] = v.reshape(-1)
            hit += 1
        if not hit:
            raise KeyError("NO node's weights could assign in self.graph {} vs {}".format(
                list(self.get_weights().keys()), list(weights.keys())))
        self.explore.copy_(torch.from_numpy(host))

    def assign_targets(self):
        """eval -> target for the agent and the mixer (qmix_tf.py:494-503)."""
        self.target.copy_(self.params)

    def assign_explore_agent(self):
        """eval agent -> explore agent (qmix_tf.py:505-511)."""
        self.explore.copy_(self.params[:self.agent_size])

    def save_explore_agent_weights(self, save_path):
        """The explore agent's variables as save_path + ".npz" (the reference writes a tf.train.Saver checkpoint)."""
        np.savez(save_path + ".npz", **self.get_weights())
        return save_path + ".npz"

    def restore_explorer_variable(self, model_name):
        """Load every explore-agent variable from a file of save_explore_agent_weights (with or without ".npz")."""
        path = model_name if model_name.endswith(".npz") else model_name + ".npz"
        with np.load(path) as f:
            stored = {k: f[k] for k in f.files}
        missing = [k for k in self.get_weights() if k not in stored]
        if missing:
            raise KeyError("update {} error: not in {}".format(missing[0], path))
        self.set_weights(stored)

    # ---- acting -----------------------------------------------------------------------------------------------------
    def reset_hidden_state(self):
        self.hidden.zero_()

    def infer_actions(self, agent_inputs):
        """Q values [1, n_agents, n_actions] of agent_inputs [1, 1, n_agents, obs_shape]; the hidden state stays on the
        device between calls."""
        x = np.asarray(agent_inputs, dtype=np.float32).reshape(self.n_agents, self.obs_shape)
        io = self._io
        stage_h2d(io["obs1"], x, np.float32)
        check(getattr(capi.lib(), self._native + "_infer")(self.handle, _ptr(self.explore), _ptr(io["obs1"]), _ptr(self.hidden),
                                                           _ptr(io["q1"]), 1 if self.use_graph else 0, stream_ptr()))
        return io["q1"].cpu().numpy().reshape(1, self.n_agents, self.n_actions)

    def reset_act_state(self, envs=None):
        """Zero hidden state and no last action for the environment slots `envs` (all when None); the Philox step counters
        keep running, so a slot's next episode draws new numbers."""
        idx = slice(None) if envs is None else torch.as_tensor(np.asarray(envs, np.int64).reshape(-1), device=self.device)
        self.act_hidden[idx] = 0.0
        self.act_last[idx] = -1

    def _act_args(self, N, epsilon, uniforms):
        """Checked n_envs, epsilon [N] and uniforms (None or [N, 2, n]) as host float64 arrays."""
        if not 1 <= N <= self.act_envs:
            raise ValueError("{} environments, act_envs is {}".format(N, self.act_envs))
        eps = np.broadcast_to(np.asarray(epsilon, np.float64), (N,))
        if uniforms is not None:
            uniforms = np.asarray(uniforms, np.float64)
            if uniforms.shape != (N, 2, self.n_agents):
                raise ValueError("uniforms: shape {} != {}".format(uniforms.shape, (N, 2, self.n_agents)))
        return eps, uniforms

    def act(self, obs, avail, reset, epsilon, uniforms=None):
        """One step of N <= act_envs environments (environment e in slot e) -> host int32 actions [N, n_agents]: obs
        [N, n_agents, act_obs_dim], avail [N, n_agents, n_actions] integer action weights (0: unavailable), reset [N]
        (True: the episode starts, zero hidden state and no last action), epsilon (scalar or [N]) and uniforms
        ([N, 2, n_agents] float64, None: Philox draws on the device).  The agent inputs, the network and the selector run
        on the device (act_device); ValueError before any launch for a wrong shape or dtype, a negative weight or a row
        without an available action (the host selector's np.random.choice fails there too)."""
        obs = np.asarray(obs)
        N = obs.shape[0] if obs.ndim == 3 else -1
        n, A = self.n_agents, self.n_actions
        if obs.shape != (N, n, self.act_obs_dim):
            raise ValueError("obs: shape {} is not [N, {}, {}]".format(obs.shape, n, self.act_obs_dim))
        av = np.asarray(avail)
        if av.shape != (N, n, A) or not (np.issubdtype(av.dtype, np.integer) or av.dtype == np.bool_):
            raise ValueError("avail: integer [{}, {}, {}] expected, got {} {}".format(N, n, A, av.dtype, av.shape))
        if np.any(av < 0) or np.any(av.astype(np.int64).sum(-1) <= 0):
            raise ValueError("avail: every row needs non-negative weights and an available action")
        if np.any(av > np.iinfo(np.int32).max):
            raise ValueError("avail: weights must fit in int32")
        rs = np.asarray(reset)
        if rs.shape != (N,):
            raise ValueError("reset: shape {} != ({},)".format(rs.shape, N))
        eps, uniforms = self._act_args(N, epsilon, uniforms)
        io = self._act_io
        stage_h2d(io["obs"][:N], obs, np.float32)
        stage_h2d(io["avail"][:N], av, np.int32)
        stage_h2d(io["reset"][:N], rs.astype(bool), np.int32)
        stage_h2d(io["epsilon"][:N], eps, np.float64)
        if uniforms is not None:
            stage_h2d(io["uniforms"][:N], uniforms, np.float64)
        out = self.act_device(io["obs"][:N], io["avail"][:N], io["reset"][:N], io["epsilon"][:N],
                              None if uniforms is None else io["uniforms"][:N], out=io["actions"][:N])
        return out.cpu().numpy()

    def act_device(self, obs, avail, reset, epsilon, uniforms=None, out=None):
        """act on contiguous device tensors (obs float32 [N, n_agents, act_obs_dim], avail int32 [N, n_agents, n_actions],
        reset int32 [N], epsilon float64 [N], uniforms float64 [N, 2, n_agents] or None) -> the int32 [N, n_agents] device
        tensor `out` (default: the model's own, overwritten by the next call).  Shapes and dtypes are checked (ValueError);
        the weights are not read on the host: a row without an available action gets an action that means nothing.  The
        Q values stay in fc2's output tensor, rows e n_agents + a."""
        N = obs.shape[0] if obs.dim() == 3 else -1
        n, A = self.n_agents, self.n_actions
        want = [("obs", obs, (N, n, self.act_obs_dim), torch.float32), ("avail", avail, (N, n, A), torch.int32),
                ("reset", reset, (N,), torch.int32), ("epsilon", epsilon, (N,), torch.float64)]
        if uniforms is not None:
            want.append(("uniforms", uniforms, (N, 2, n), torch.float64))
        if out is None:
            out = self._act_io["actions"][:max(N, 0)]
        want.append(("out", out, (N, n), torch.int32))
        dev = self.act_hidden.device
        for name, t, shape, dt in want:
            if tuple(t.shape) != shape or t.dtype != dt or t.device != dev or not t.is_contiguous():
                raise ValueError("{}: contiguous {} {} on {} expected, got {} {} on {}".format(name, dt, shape, dev, t.dtype,
                                                                                           tuple(t.shape), t.device))
        self._act_args(N, 0.0, None)
        if uniforms is None and self._act_seed is None:
            self._act_seed = int(self._init_rng.integers(0, 2 ** 63))
        check(getattr(capi.lib(), self._native + "_act")(
            self.handle, _ptr(self.explore), N, int(self.obs_last_action), int(self.obs_agent_id), _ptr(obs), _ptr(avail), _ptr(reset),
            _ptr(epsilon), _ptr(uniforms), self._act_seed or 0, _ptr(self.act_counter), _ptr(self.act_hidden), _ptr(self.act_last),
            _ptr(out), 1 if self.use_graph else 0, stream_ptr()))
        return out

    # ---- training ---------------------------------------------------------------------------------------------------
    def _train_buffers(self):
        if self._bufs is None:
            B, L, n, A, dev = self._B, self._L, self.n_agents, self.n_actions, self.device
            f32 = dict(dtype=torch.float32, device=dev)
            self._bufs = dict(obs=torch.empty(B, L + 1, n, self.obs_shape, **f32),
                              seq_len=torch.empty(B * n, dtype=torch.int32, device=dev),
                              avail=torch.empty(B, L + 1, n, A, **f32),
                              actions=torch.empty(B, L, n, dtype=torch.int32, device=dev),
                              state=torch.empty(B, L, self.state_dim, **f32), next_state=torch.empty(B, L, self.state_dim, **f32),
                              reward=torch.empty(B, L, **f32), terminated=torch.empty(B, L, **f32), mask=torch.empty(B, L, **f32),
                              loss=torch.zeros(1, **f32))
        return self._bufs

    def _agent_batch(self, train_obs_len, actions):
        """A train call's sequence lengths [batch_size * n_agents] and actions [batch_size, episode_limit, n_agents],
        checked -> (seq_len, actions)."""
        B, L, n, A = self._B, self._L, self.n_agents, self.n_actions
        seq_len = np.asarray(train_obs_len).reshape(-1)
        if seq_len.size != B * n or np.any(seq_len < 0) or np.any(seq_len > L + 1):
            raise ValueError("train_obs_len: {} lengths in [0, {}] expected".format(B * n, L + 1))
        act = np.asarray(actions).reshape(B, L, n)
        if np.any(act < 0) or np.any(act >= A):
            raise ValueError("actions must be in [0, {})".format(A))
        return seq_len, act

    def train(self, batch_trajectories, train_obs_len, avail_actions, actions, cur_stats, target_stats, rewards, terminated, mask):
        """qmix_tf.py:546-589: one RMSProp step on a [batch_size, episode_limit (+1), ...] batch -> loss."""
        if self.opt is None:
            raise RuntimeError("QMixModel.train needs the train scene")
        seq_len, act = self._agent_batch(train_obs_len, actions)
        b = self._train_buffers()
        stage_h2d(b["obs"], batch_trajectories, np.float32)
        stage_h2d(b["seq_len"], seq_len, np.int32)
        stage_h2d(b["avail"], avail_actions, np.float32)
        stage_h2d(b["actions"], act, np.int32)
        stage_h2d(b["state"], cur_stats, np.float32)
        stage_h2d(b["next_state"], target_stats, np.float32)
        stage_h2d(b["reward"], rewards, np.float32)
        stage_h2d(b["terminated"], terminated, np.float32)
        stage_h2d(b["mask"], mask, np.float32)
        self.train_device(b)
        return float(b["loss"].cpu()[0])

    def _replay_out(self, n_loss):
        """[n_loss losses | max_t_filled as int32] side by side, for one download per train_replay."""
        if getattr(self, "_rout", None) is None:
            self._rout = torch.zeros(n_loss + 1, dtype=torch.float32, device=self.device)
        return self._rout

    def train_replay(self, replay, ids):
        """QMixAlg.train's step on the episodes `ids` of a DeviceEpisodeReplay (xtb_qmix_replay_train, graph-replayed
        when the model uses graphs): one staged upload of the ids, the batch gathered into _train_buffers() and the
        step of train(), one download -> (loss, max_t_filled)."""
        if self.opt is None:
            raise RuntimeError("QMixModel.train_replay needs the train scene")
        b = self._train_buffers()
        out = self._replay_out(1)
        bt = capi.QmixBatch()
        for k in ("obs", "seq_len", "avail", "actions", "state", "next_state", "reward", "terminated", "mask"):
            setattr(bt, k, b[k].data_ptr())
        ids = np.ascontiguousarray(ids, np.int32)
        check(capi.lib().xtb_qmix_replay_train(replay.handle, self.handle, self.opt.handle, _ptr(self.target), len(ids), ids.ctypes.data,
                                               C.byref(bt), _ptr(out[:1]), _ptr(out[1:]), 1 if self.use_graph else 0, stream_ptr()))
        host = out.cpu().numpy()
        return float(host[0]), int(host[1:].view(np.int32)[0])

    def train_device(self, b):
        """xtb_qmix_train on the device tensors of _train_buffers(); the loss lands in b["loss"]."""
        bt = capi.QmixBatch()
        for k in ("obs", "seq_len", "avail", "actions", "state", "next_state", "reward", "terminated", "mask"):
            setattr(bt, k, b[k].data_ptr())
        check(capi.lib().xtb_qmix_train(self.handle, self.opt.handle, _ptr(self.target), C.byref(bt), _ptr(b["loss"]),
                                        1 if self.use_graph else 0, stream_ptr()))
