"""MuzeroModel / MuzeroCnn / MuzeroMlp on the CUDA engine (xt/model/muzero/muzero_model.py, muzero_cnn.py, muzero_mlp.py).

The representation, dynamics and prediction networks are three engine nets bound to consecutive slices of one flat
parameter buffer (and one gradient buffer) in MuzeroBase's Keras weight-list order, trained by one Adam.  The unrolled
training step, the support projections, the inference calls and the tree search over many observations at once
(search / search_device) run in libxtb200 (xtb_muzero_*)."""
import ctypes as C
import math
import os
import typing
from types import SimpleNamespace
from typing import List

import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, Net, _ptr, stage_h2d, stream_ptr
from ..registry import Registers, import_config
from . import archs
from .base import XTModel, check_keep_model, glorot_uniform_

# xt/model/muzero/default_config.py
HIDDEN1_UNITS = 64
HIDDEN2_UNITS = 4
LR = 1e-3
td_step = 5
max_value = 500
HIDDEN_OUT = 256

WEIGHT_DECAY = 1e-4   # muzero_model.py:58


def value_compression(value):
    """muzero_utils.py:38-40: h(x) = sign(x)(sqrt(|x| + 1) - 1) + 0.001 x."""
    return np.sign(value) * (np.sqrt(np.abs(value) + 1) - 1) + 0.001 * value


def value_decompression(value):
    """muzero_utils.py:43-47: the closed-form inverse of h."""
    return np.sign(value) * (((np.sqrt(1 + 4 * 0.001 * (np.abs(value) + 1 + 0.001)) - 1) / (2 * 0.001)) ** 2 - 1)


def support_size(vmin, vmax):
    """muzero_model.py:47-52: ceil(h(max - min)) + 1."""
    return int(math.ceil(value_compression(vmax - vmin))) + 1


class NetworkOutput(typing.NamedTuple):
    """muzero_model.py:242-246."""
    value: float
    reward: float
    policy: List[int]
    hidden_state: List[float]


class MuzeroModel(XTModel):
    """Shared body of MuzeroCnn / MuzeroMlp.  Sub-classes implement build_archs()."""

    def __init__(self, model_info):
        model_config = model_info.get("model_config", None) or {}
        import_config(globals(), model_config)
        self.state_dim = model_info["state_dim"]
        self.action_dim = model_info["action_dim"]
        self.reward_min = model_config.get("reward_min", -300)
        self.reward_max = model_config.get("reward_max", 300)
        self.reward_support_size = support_size(self.reward_min, self.reward_max)
        self.value_min = model_config.get("value_min", 0)
        self.value_max = model_config.get("value_max", 60000)
        self.value_support_size = support_size(self.value_min, self.value_max)
        self.obs_type = model_config.get("obs_type", "float32")
        if self.obs_type not in ("float32", "uint8", "int8"):
            raise ValueError("MuZero obs_type {!r} is not supported (float32, uint8 or int8)".format(self.obs_type))
        self.td_step = int(td_step)
        self.learning_rate = LR
        self.max_batch = int(model_config.get("max_batch", 1024))
        super().__init__(model_info)

    def build_archs(self):
        raise NotImplementedError

    def create_model(self, model_info):
        rep_a, dyn_a, pred_a = self.build_archs()
        if rep_a["input_dtype"] == "uint8":
            # MuzeroCnn casts the obs placeholder (dtype obs_type) to float and divides by 255: a float frame as it is,
            # an int8 placeholder fed uint8 bytes as their two's-complement values
            rep_a = dict(rep_a, input_dtype=self.obs_type)
        elif self.obs_type != "float32":
            raise ValueError("obs_type {!r}: this model reads float observations".format(self.obs_type))
        B, K = self.max_batch, self.td_step
        self.rep = Net(rep_a, max_batch=B, device=self.device)
        self.dyn = Net(dyn_a, max_batch=B, device=self.device)
        self.pred = Net(pred_a, max_batch=(K + 1) * B, device=self.device)
        nets = (self.rep, self.dyn, self.pred)
        # each slice starts 256-byte aligned (the tensor-core weight refresh reads 16-byte pieces); the gaps stay zero
        offs = [0]
        for n in nets[:-1]:
            offs.append((offs[-1] + n.n_params + 63) // 64 * 64)
        self.n_params = offs[-1] + self.pred.n_params
        self.params = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
        self.grads = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
        self._dyn_grads = torch.zeros(self.dyn.n_params, dtype=torch.float32, device=self.device)
        for n, off in zip(nets, offs):
            g = self._dyn_grads if n is self.dyn else self.grads[off:off + n.n_params]
            n.bind_to(self.params[off:off + n.n_params], g)
        for n in nets:
            glorot_uniform_(n, self._init_rng)
        # the l2 term of build_train_graph is taken of get_weights() arrays: a constant of the initial weights, no gradient
        self.weight_decay_loss = float(WEIGHT_DECAY * sum(0.5 * np.sum(np.square(w, dtype=np.float64)) for w in self.get_weights()))
        flat = SimpleNamespace(params=self.params, n_params=self.n_params, device=self.device,
                               segment_offsets=lambda: [0, self.n_params])
        self.opt = Adam(flat, self.learning_rate, eps=1e-8, clip_mode=capi.CLIP_NONE, clip=0.0)
        desc = capi.MuzeroDesc()
        desc.unroll = K
        desc.rep_h = self.rep.tid[rep_a["outputs"][0]]
        desc.dyn_h, desc.dyn_r = (self.dyn.tid[n] for n in dyn_a["outputs"])
        desc.pred_p, desc.pred_v = (self.pred.tid[n] for n in pred_a["outputs"])
        desc.value_min, desc.value_max = float(self.value_min), float(self.value_max)
        desc.reward_min, desc.reward_max = float(self.reward_min), float(self.reward_max)
        self.handle = C.c_void_p()
        with torch.cuda.device(self.device):
            check(capi.lib().xtb_muzero_create(self.rep.handle, self.dyn.handle, self.pred.handle, C.byref(desc), B,
                                               C.byref(self.handle)))
        self.hidden_dim = self.rep.lib.xtb_net_tensor_size(self.rep.handle, desc.rep_h)
        self._bytes = rep_a["input_dtype"] in ("uint8", "int8")     # frames travel as bytes either way
        self._obs_dt = torch.uint8 if self._bytes else torch.float32
        self._np_dt = np.uint8 if self._bytes else np.float32
        self._bufs = {}
        self.net = self.rep
        return self.rep

    def __del__(self):
        try:
            self._drop_tree()
            if getattr(self, "handle", None) and self.handle.value:
                capi.lib().xtb_muzero_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:
            pass

    # ---- weights: a Keras list in MuzeroBase order (representation, dynamics, prediction) --------------------------
    def _tables(self):
        out = []
        for n in (self.rep, self.dyn, self.pred):
            base = n.params.data_ptr() - self.params.data_ptr()
            for name, (off, shape) in n.ptable.items():
                out.append((base // 4 + off, shape))
        return out

    def get_weights(self):
        host = self.params.detach().cpu().numpy()
        return [host[o:o + int(np.prod(s))].reshape(s).copy() for o, s in self._tables()]

    def set_weights(self, weights):
        tables = self._tables()
        if len(weights) != len(tables):
            raise ValueError("expected {} weight arrays, got {}".format(len(tables), len(weights)))
        host = self.params.detach().cpu().numpy().copy()
        for (o, s), w in zip(tables, weights):
            w = np.asarray(w, dtype=np.float32)
            if tuple(w.shape) != tuple(s):
                raise ValueError("weight shape {} != {}".format(w.shape, s))
            host[o:o + w.size] = w.reshape(-1)
        self.params.copy_(torch.from_numpy(host))
        for n in (self.rep, self.dyn, self.pred):
            n.params_changed()

    def save_model(self, file_name):
        """The weight list as .npz (arr_0, arr_1, ... in list order); the reference writes Keras .h5."""
        if self.max_to_keep > -1:
            check_keep_model(os.path.dirname(file_name), self.max_to_keep)
        np.savez(file_name + ".npz", *self.get_weights())
        return file_name + ".npz"

    def load_model(self, model_name, by_name=False):
        f = np.load(model_name)
        self.set_weights([f["arr_%d" % i] for i in range(len(f.files))])

    # ---- device buffers -------------------------------------------------------------------------------------------
    def _buffers(self, n):
        b = self._bufs.get(n)
        if b is None:
            dev, K, A = self.device, self.td_step, self.action_dim
            b = dict(obs=torch.empty((n,) + tuple(self.state_dim), dtype=self._obs_dt, device=dev),
                     action=torch.empty(n, K, dtype=torch.int32, device=dev),
                     tv=torch.empty(n, K + 1, dtype=torch.float32, device=dev),
                     tr=torch.empty(n, K + 1, dtype=torch.float32, device=dev),
                     tp=torch.empty(n, K + 1, A, dtype=torch.float32, device=dev),
                     loss=torch.zeros(1, dtype=torch.float32, device=dev),
                     value=torch.empty(n, dtype=torch.float32, device=dev),
                     reward=torch.empty(n, dtype=torch.float32, device=dev),
                     policy=torch.empty(n, A, dtype=torch.float32, device=dev),
                     hidden=torch.empty(n, self.hidden_dim, dtype=torch.float32, device=dev),
                     hidden_r=torch.empty(n, self.hidden_dim, dtype=torch.float32, device=dev),
                     hid_in=torch.empty(n, self.hidden_dim, dtype=torch.float32, device=dev),
                     act1=torch.empty(n, dtype=torch.int32, device=dev))
            self._bufs[n] = b
        return b

    def _host_obs(self, obs):
        """Observations as the bytes / floats the device reads: an int8 model takes the two's-complement bytes of the
        values (uint8 frames pass unchanged, as np.asarray(frames, dtype=int8) reinterprets them)."""
        if self.obs_type == "int8":
            return np.ascontiguousarray(np.asarray(obs).astype(np.int8)).view(np.uint8)
        return np.ascontiguousarray(obs, self._np_dt)

    def _check_batch(self, n):
        if n < 1 or n > self.max_batch:
            raise ValueError("batch {} not in [1, max_batch={}]".format(n, self.max_batch))

    # ---- training -------------------------------------------------------------------------------------------------
    def train_device(self, obs, action, target_value, target_reward, target_policy, n, loss_buf, value_buf=None):
        """One training step on device tensors (see xtb_muzero_train); loss_buf[0] = the reported loss, value_buf [n] (if
        given) = value_inference of obs after the update."""
        self._check_batch(n)
        bt = capi.MuzeroBatch()
        bt.obs, bt.action = obs.data_ptr(), action.data_ptr()
        bt.target_value, bt.target_reward, bt.target_policy = target_value.data_ptr(), target_reward.data_ptr(), target_policy.data_ptr()
        bt.unroll = self.td_step
        check(capi.lib().xtb_muzero_train(self.handle, self.opt.handle, C.byref(bt), int(n), float(self.weight_decay_loss),
                                          _ptr(loss_buf), _ptr(value_buf), 1 if self.use_graph else 0, stream_ptr()))
        return loss_buf

    def train(self, state, label):
        """muzero_model.py:154-169: state = [obs, action [B, K], loss_weights (unused)], label = [target_value [B, K+1],
        target_reward [B, K+1], target_policy [B, K+1, A]] -> loss."""
        return self.train_and_values(state[0], state[1], label[0], label[1], label[2], values=False)[0]

    def train_and_values(self, obs, action, target_value, target_reward, target_policy, values=True):
        """Upload one host minibatch through the staged pinned copy (xtb_copy_h2d_staged) and run one step ->
        (loss, the post-update value of every observation as float64, or None)."""
        obs = self._host_obs(obs)
        n = obs.shape[0]
        self._check_batch(n)
        b = self._buffers(n)
        stage_h2d(b["obs"], obs, self._np_dt)
        stage_h2d(b["action"], np.asarray(action), np.int32)
        stage_h2d(b["tv"], np.asarray(target_value), np.float32)
        stage_h2d(b["tr"], np.asarray(target_reward), np.float32)
        stage_h2d(b["tp"], np.asarray(target_policy), np.float32)
        self.train_device(b["obs"], b["action"], b["tv"], b["tr"], b["tp"], n, b["loss"], b["value"] if values else None)
        loss = float(b["loss"].cpu()[0])
        return loss, (b["value"].cpu().numpy().astype(np.float64) if values else None)

    # ---- inference ------------------------------------------------------------------------------------------------
    def initial_inference_batch(self, obs, n):
        """Batched initial_inference on device observations: (value [n], policy [n, A], hidden [n, H]) device tensors.
        They are buffers of this model, per batch size: the next initial_inference_batch of the same size overwrites them
        (clone what must outlive it)."""
        self._check_batch(n)
        b = self._buffers(n)
        check(capi.lib().xtb_muzero_initial_inference(self.handle, _ptr(obs), int(n), _ptr(b["hidden"]), _ptr(b["value"]),
                                                      _ptr(b["policy"]), 1 if self.use_graph else 0, stream_ptr()))
        return b["value"], b["policy"], b["hidden"]

    def recurrent_inference_batch(self, hidden, action, n):
        """Batched recurrent_inference on device hidden states [n, H] and actions [n] (int32): (value [n], reward [n],
        policy [n, A], next hidden [n, H]) device tensors, overwritten by the next call of the same size (its own buffers,
        apart from initial_inference_batch's hidden states, so those may be fed back in)."""
        self._check_batch(n)
        b = self._buffers(n)
        check(capi.lib().xtb_muzero_recurrent_inference(self.handle, _ptr(hidden), _ptr(action), int(n), _ptr(b["hidden_r"]),
                                                        _ptr(b["reward"]), _ptr(b["value"]), _ptr(b["policy"]),
                                                        1 if self.use_graph else 0, stream_ptr()))
        return b["value"], b["reward"], b["policy"], b["hidden_r"]

    def initial_inference(self, input_data):
        """muzero_model.py:74-82: NetworkOutput(value, 0, policy, hidden) of sample 0."""
        obs = self._host_obs(input_data)
        n = obs.shape[0]
        self._check_batch(n)
        b = self._buffers(n)
        stage_h2d(b["obs"], obs, self._np_dt)
        value, policy, hidden = self.initial_inference_batch(b["obs"], n)
        return NetworkOutput(float(value[0].cpu()), 0, policy[0].cpu().numpy(), hidden[0].cpu().numpy())

    def recurrent_inference(self, hidden_state, action):
        """muzero_model.py:84-96: NetworkOutput(value, reward, policy, hidden) for one hidden state and action."""
        b = self._buffers(1)
        stage_h2d(b["hid_in"], np.asarray(hidden_state).reshape(1, -1), np.float32)
        stage_h2d(b["act1"], np.asarray([int(action)]), np.int32)
        value, reward, policy, hidden = self.recurrent_inference_batch(b["hid_in"], b["act1"], 1)
        return NetworkOutput(float(value[0].cpu()), float(reward[0].cpu()), policy[0].cpu().numpy(), hidden[0].cpu().numpy())

    # ---- tree search ----------------------------------------------------------------------------------------------
    def _search_tree(self, n, num_simulations):
        """The tree scratch for n trees of num_simulations simulations: created on first use, grown (never shrunk) when
        a call needs more trees or simulations than it holds."""
        envs, sims = getattr(self, "_tree_size", (0, 0))
        if n > envs or num_simulations > sims:
            envs, sims = max(n, envs), max(num_simulations, sims)
            self._drop_tree()
            tree = C.c_void_p()
            with torch.cuda.device(self.device):
                check(capi.lib().xtb_muzero_tree_create(self.handle, envs, sims, C.byref(tree)))
            self._tree, self._tree_size = tree, (envs, sims)
        return self._tree

    def _drop_tree(self):
        tree = getattr(self, "_tree", None)
        if tree is not None and tree.value:
            capi.lib().xtb_muzero_tree_destroy(tree)
        self._tree, self._tree_size = None, (0, 0)

    def _search_buffers(self, n):
        """[n] float64 root values followed by the [n, A] int32 visit counts in one device block (one download), and the
        [n, A] float64 noise."""
        key = ("search", n)
        b = self._bufs.get(key)
        if b is None:
            A = self.action_dim
            out = torch.empty(n + (n * A + 1) // 2, dtype=torch.float64, device=self.device)
            b = dict(out=out, root_value=out[:n], counts=out[n:].view(torch.int32)[:n * A].view(n, A),
                     noise=torch.empty(n, A, dtype=torch.float64, device=self.device))
            self._bufs[key] = b
        return b

    def search_device(self, obs, n, num_simulations, noise=None, visit_counts=None, root_value=None, pb_c_base=19652,
                      pb_c_init=1.25, discount=0.997, exploration_frac=0.25):
        """Mcts.run_mcts (xt/agent/muzero/mcts.py) over n device observations at once, one tree each (xtb_muzero_search):
        -> (visit_counts [n, A] int32, root_value [n] float64) device tensors.  noise [n, A] float64 (device) mixes
        into the root priors as the reference's add_exploration_noise.  Without visit_counts / root_value the results go
        to buffers of this model, per n, that the next search of the same size overwrites."""
        self._check_batch(n)
        b = self._search_buffers(n)
        visit_counts = b["counts"] if visit_counts is None else visit_counts
        root_value = b["root_value"] if root_value is None else root_value
        tree = self._search_tree(n, int(num_simulations))
        check(capi.lib().xtb_muzero_search(self.handle, tree, _ptr(obs), int(n), int(num_simulations), _ptr(noise),
                                           float(pb_c_base), float(pb_c_init), float(discount), float(exploration_frac),
                                           _ptr(visit_counts), _ptr(root_value), 1 if self.use_graph else 0, stream_ptr()))
        return visit_counts, root_value

    def search(self, obs, num_simulations, noise=None, **kw):
        """search_device on host observations [n, ...] (and host noise [n, A]): staged uploads, one search, one download
        -> (visit_counts [n, A] int32, root_value [n] float64) numpy arrays."""
        obs = self._host_obs(obs)
        n = obs.shape[0]
        self._check_batch(n)
        b, sb = self._buffers(n), self._search_buffers(n)
        stage_h2d(b["obs"], obs, self._np_dt)
        if noise is not None:
            stage_h2d(sb["noise"], np.asarray(noise), np.float64)
        self.search_device(b["obs"], n, num_simulations, sb["noise"] if noise is not None else None, **kw)
        host = sb["out"].cpu().numpy()
        A = self.action_dim
        return host[n:].view(np.int32)[:n * A].reshape(n, A).copy(), host[:n].copy()

    def value_inference(self, input_data):
        """muzero_model.py:228-239: the scalar value of every observation (any count: max_batch rows per call)."""
        obs = self._host_obs(input_data)
        out = []
        for s in range(0, obs.shape[0], self.max_batch):
            part = obs[s:s + self.max_batch]
            n = part.shape[0]
            b = self._buffers(n)
            stage_h2d(b["obs"], part, self._np_dt)
            check(capi.lib().xtb_muzero_initial_inference(self.handle, _ptr(b["obs"]), int(n), None, _ptr(b["value"]), None,
                                                          1 if self.use_graph else 0, stream_ptr()))
            out.append(b["value"].cpu().numpy().astype(np.float64))
        return np.concatenate(out) if out else np.zeros(0)


@Registers.model
class MuzeroCnn(MuzeroModel):
    """MuzeroCnn (xt/model/muzero/muzero_cnn.py:31-67): PpoCnn-style conv trunk to a HIDDEN_OUT-wide hidden state."""

    def build_archs(self):
        return archs.muzero_cnn(self.state_dim, self.action_dim, self.value_support_size, self.reward_support_size, HIDDEN_OUT)


@Registers.model
class MuzeroMlp(MuzeroModel):
    """MuzeroMlp (xt/model/muzero/muzero_mlp.py:30-63): HIDDEN1_UNITS dense layers, a HIDDEN2_UNITS-wide hidden state."""

    def build_archs(self):
        return archs.muzero_mlp(self.state_dim, self.action_dim, self.value_support_size, self.reward_support_size,
                                HIDDEN1_UNITS, HIDDEN2_UNITS)
