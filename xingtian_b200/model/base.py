"""XTModel base: the reference's model surface (xt/model/model.py:30-136) over the CUDA engine."""
import glob
import math
import os
from collections import OrderedDict

import numpy as np
import torch

from ..engine import Net, require_cuda


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


def check_keep_model(model_path, keep_num):
    """xt/model/model.py:125-132."""
    target_file = glob.glob(os.path.join(model_path, "actor*"))
    if len(target_file) > keep_num:
        to_rm_model = sorted(target_file, reverse=True)[keep_num:]
        for item in to_rm_model:
            os.remove(item)
