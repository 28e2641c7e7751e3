"""XTModel base: the reference's model surface (xt/model/model.py:30-136) over the CUDA engine."""
import ctypes as C
import glob
import math
import os
from collections import OrderedDict

import numpy as np
import torch

from ..capi import check
from ..engine import Net, _ptr, require_cuda, stream_ptr


def glorot_uniform_(net, rng):
    """Keras default initialisation: glorot_uniform kernels, zero biases (and zero pi_logstd, ppo.py:77)."""
    host = np.zeros(net.n_params, np.float32)
    for name, (off, shape) in net.ptable.items():
        if not name.endswith("/kernel"):
            continue
        if len(shape) == 4:
            rf = shape[0] * shape[1]
            fan_in, fan_out = rf * shape[2], rf * shape[3]
        else:
            fan_in, fan_out = shape
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        host[off:off + int(np.prod(shape))] = rng.uniform(-lim, lim, size=int(np.prod(shape))).astype(np.float32)
    net.params.copy_(torch.from_numpy(host))
    net.params_changed()


class XTModel(object):
    """Model base class (xt/model/model.py:30-136).

    Sub-classes implement ``create_model`` (build the device network), ``predict`` and ``train``.
    Weights travel as an OrderedDict{tf variable name -> ndarray} and are stored as ``.npz``
    exactly like TFVariables (xt/model/tf_utils.py:99-144)."""

    def __init__(self, model_info):
        require_cuda()
        model_config = model_info.get("model_config") or {}
        seed = model_config.get("init_seed")
        # the generator every initial weight is drawn from (not the global np.random stream)
        self._init_rng = np.random.default_rng(seed) if seed is not None else np.random.default_rng()
        self.use_graph = bool(model_config.get("use_cuda_graph", True))
        self.actor_var = None
        self._summary = model_info.get("summary", False)
        self.model_format = model_info.get("model_format")
        self.max_to_keep = model_info.get("max_to_keep", 100)
        self.device = torch.device(model_info.get("device", "cuda:%d" % torch.cuda.current_device()))
        if self.device.type != "cuda" or (self.device.index is not None and self.device.index != torch.cuda.current_device()):
            # native calls run on the current device's stream and the staging ring lives on the device of its first use
            raise ValueError("model device {} is not the current CUDA device {}: call torch.cuda.set_device first".format(
                self.device, torch.cuda.current_device()))
        self.net = None
        self.model = self.create_model(model_info)
        if "init_weights" in model_info:
            model_name = model_info["init_weights"]
            try:
                self.load_model(model_name)
                print("load weight: {} success.".format(model_name))
            except BaseException:
                print("load weight: {} failed!".format(model_name))

    def create_model(self, model_info):
        raise NotImplementedError

    def seeded_net(self, arch, max_batch):
        """A Net of `arch` with glorot_uniform_ weights from the model's init generator; the observations the model
        takes (`_obs_dt` on the device, `_np_dt` on the host) are the arch's input dtype."""
        net = Net(arch, max_batch=max_batch, device=self.device)
        glorot_uniform_(net, self._init_rng)
        u8 = arch["input_dtype"] == "uint8"
        self._obs_dt, self._np_dt = (torch.uint8, np.uint8) if u8 else (torch.float32, np.float32)
        return net

    def predict(self, state):
        raise NotImplementedError

    def train(self, state, label):
        raise NotImplementedError

    def set_weights(self, weights):
        """xt/model/model.py:84-87."""
        self.net.set_weights(weights)

    def get_weights(self):
        """xt/model/model.py:89-92."""
        return self.net.get_weights()

    def save_model(self, file_name):
        """xt/model/model.py:99-114: numpy .npz keyed by variable name; keep-last-N."""
        if self.max_to_keep > -1:
            check_keep_model(os.path.dirname(file_name), self.max_to_keep)
        np.savez(file_name + ".npz", **self.get_weights())
        return file_name + ".npz"

    def load_model(self, model_name, by_name=False):
        """xt/model/model.py:116-122 / tf_utils.py:135-144."""
        np_file = np.load(model_name)
        self.set_weights(OrderedDict(**np_file))


class PolicyActor(object):
    """The native sampling calls of an actor-critic policy (PPO, ImpalaCnnOpt).  The subclass sets `net`, `device`,
    `use_graph`, `state_dim`, `action_dim`, `_obs_dt` (observation dtype) and the heads: `pi_t` (logits, or the
    DiagGaussian mean), `v_t` (value) and `ls_t` (0 for Categorical, else the DiagGaussian's logstd tensor)."""

    predict_head = False    # the host predict also copies the pi head's output (ImpalaCnnOpt.predict returns the logits)

    def _init_sampling(self):
        """Draw the Philox seed of every sampling call (one global np.random draw) and reset the counters."""
        self._sample_seed = int(np.random.randint(0, 2 ** 31 - 1))
        self._sample_offset = 0      # host counter of the calls that take their offset from the host
        self._offset_dev = None      # device counter of rollout inference and host predict, created at first use
        self._predict_ios = {}

    def _offset(self):
        if self._offset_dev is None:
            self._offset_dev = torch.zeros(1, dtype=torch.int64, device=self.device)
        return self._offset_dev

    def _predict_io(self, batch):
        """Persistent staging of the host predict: device input, one packed device / pinned output block
        [action | logp | value] (a DiagGaussian's action is A rows) and, with predict_head, a pinned [batch, A] block for
        the pi head, so a call is 1 H2D + 1 graph launch + 1 D2H."""
        io = self._predict_ios.get(batch)
        if io is None:
            rows = (self.action_dim if self.ls_t else 1) + 2
            out_dev = torch.empty(rows, batch, dtype=torch.float32, device=self.device)
            head = torch.empty(batch, self.action_dim, dtype=torch.float32).pin_memory() if self.predict_head else None
            io = dict(obs=torch.empty((batch,) + tuple(self.state_dim), dtype=self._obs_dt, device=self.device),
                      out_dev=out_dev, act=out_dev[0].view(torch.int32), logp=out_dev[rows - 2], val=out_dev[rows - 1],
                      pin_out=torch.empty(rows, batch, dtype=torch.float32).pin_memory(), pin_head=head)
            io["obs_ptr"], io["out_dev_ptr"], io["pin_out_ptr"] = _ptr(io["obs"]), _ptr(out_dev), _ptr(io["pin_out"])
            io["pin_out_np"] = io["pin_out"].numpy()
            self._predict_ios[batch] = io
        return io

    def _predict_host(self, state):
        """Staged H2D of `state` -> graphed forward + sampling -> packed D2H (+ the pi head) -> stream sync, in one
        native call; returns the IO block holding the results."""
        batch = state.shape[0]
        io = self._predict_io(batch)
        self.net.ensure_batch(batch)
        check(self.net.lib.xtb_ppo_predict_host(self.net.handle, state.ctypes.data, state.nbytes, io["obs_ptr"], batch,
                                                self.pi_t, self.v_t, self.ls_t, C.c_uint64(self._sample_seed), _ptr(self._offset()),
                                                io["out_dev_ptr"], io["pin_out_ptr"], _ptr(io["pin_head"]),
                                                1 if self.use_graph else 0, stream_ptr()))
        return io

    def _draw(self, batch, action, logp, noise=None):
        """Sample `batch` actions from the pi head of the last forward into the device tensors action / logp: Categorical
        logits, or with ls_t the DiagGaussian mean and the pi_logstd weights.  `noise` (device [batch, A]: uniforms, or
        normals for a DiagGaussian) replaces the Philox draws of (seed, `_sample_offset`); the host counter advances once."""
        net = self.net
        pi, seed, off = _ptr(net.tensor(net.names[self.pi_t])), C.c_uint64(self._sample_seed), C.c_uint64(self._sample_offset)
        if self.ls_t:
            check(net.lib.xtb_diag_gaussian_sample(pi, _ptr(net.view(net.names[self.ls_t])), batch, self.action_dim, _ptr(noise),
                                                   seed, off, _ptr(action), _ptr(logp), stream_ptr()))
        else:
            check(net.lib.xtb_categorical_sample(pi, batch, self.action_dim, _ptr(noise), seed, off, _ptr(action), _ptr(logp),
                                                 stream_ptr()))
        self._sample_offset += 1

    def rollout_infer_device(self, obs_dev, step_idx, n_env, n_step, action, logp, value):
        """n_step batched policy evaluations on device-resident observations as ONE CUDA graph (the learner-side
        replacement of the explorers' per-step predict calls): time-major action / logp / value [n_step, n_env] (a
        DiagGaussian's action f32 [n_step, n_env, A]); the pi head of the last step stays in net.tensor."""
        self.net.ensure_batch(n_env)
        check(self.net.lib.xtb_ppo_rollout_infer(self.net.handle, _ptr(obs_dev), _ptr(step_idx), int(n_env), int(n_step),
                                                 self.pi_t, self.v_t, self.ls_t, C.c_uint64(self._sample_seed),
                                                 _ptr(self._offset()), _ptr(action), _ptr(logp), _ptr(value),
                                                 1 if self.use_graph else 0, stream_ptr()))


def check_keep_model(model_path, keep_num):
    """xt/model/model.py:125-132."""
    target_file = glob.glob(os.path.join(model_path, "actor*"))
    if len(target_file) > keep_num:
        to_rm_model = sorted(target_file, reverse=True)[keep_num:]
        for item in to_rm_model:
            os.remove(item)
