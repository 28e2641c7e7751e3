"""QMixModel on the CUDA engine (xt/model/qmix/qmix_tf.py).

The reference builds five TF sub-graphs: the explore agent (one step, hidden state carried between calls), the eval and
target agents over whole episodes, and the eval and target mixers.  Here a weight set is one flat buffer
[fc1 | GRU | fc2 | mixer] in the TF variable order of the eval_agent and eval_mixer scopes: the eval set is the one the
engine nets (fc1, fc2 and the hypernetworks) are bound to and the optimiser steps, the target set and the explore agent
are buffers of the same layout.  The training step (xtb_qmix_train) and the one-step inference (xtb_qmix_infer) run in
libxtb200."""
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

    _native = "xtb_qmix"   # the native object's entry points: <_native>_infer and <_native>_destroy

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
        self.handle = C.c_void_p()
        with torch.cuda.device(dev):
            check(capi.lib().xtb_qmix_create(self.fc1.handle, self.fc2.handle, self.hyper.handle, C.byref(desc), C.byref(self.handle)))
        self._acting_state()
        return self.fc1

    def _agent_nets(self, train):
        """fc1 and fc2 for the scene's training batch and the agent's variable table -> (batch, episode limit).  The
        explore scene keeps a minimal training shape: only the one-step inference runs."""
        H, A, n = self.rnn_hidden_dim, self.n_actions, self.n_agents
        B, L = (self.batch_size, self.fix_seq_length) if train else (1, 1)
        fc1_a = dict(input_dtype="float32", state_dim=(self.obs_shape,), scale=1.0,
                     layers=[("dense", "dense", "obs", dict(n=H, act="relu"))])
        fc2_a = dict(input_dtype="float32", state_dim=(H,), scale=1.0, layers=[("dense_1", "dense", "obs", dict(n=A, act=None))])
        self.fc1 = Net(fc1_a, max_batch=B * (L + 1) * n, device=self.device)
        self.fc2 = Net(fc2_a, max_batch=B * (L + 1) * n, device=self.device)
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
        """The hidden state and the one-step inference's staging; the training buffers are made at first use."""
        n, dev = self.n_agents, self.device
        self.hidden = torch.zeros(n, self.rnn_hidden_dim, dtype=torch.float32, device=dev)
        self._io = dict(obs1=torch.empty(n, self.obs_shape, dtype=torch.float32, device=dev),
                        q1=torch.empty(n, self.n_actions, dtype=torch.float32, device=dev))
        self._bufs = None
        self.net = self.fc1

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
