"""DqnCnn / DqnMlp on the CUDA engine (xt/model/dqn/dqn_cnn.py:31-83, dqn_mlp.py:30-76)."""
import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, Net, _ptr, stream_ptr
from ..registry import Registers, import_config
from . import archs
from .base import XTModel, glorot_uniform_

# xt/model/dqn/default_config.py
HIDDEN_SIZE = 128
NUM_LAYERS = 1
LR = 0.0003


class _DqnBase(XTModel):
    clipnorm = None

    def __init__(self, model_info):
        model_config = model_info.get("model_config", None) or {}
        import_config(globals(), model_config)
        self.state_dim = model_info["state_dim"]
        self.action_dim = model_info["action_dim"]
        self.learning_rate = LR
        self.dueling = bool(model_config.get("dueling", False))
        self._init_seed = model_config.get("init_seed")
        self.use_graph = bool(model_config.get("use_cuda_graph", True))
        super().__init__(model_info)

    def build_arch(self):
        raise NotImplementedError

    def create_model(self, model_info):
        arch = self.build_arch()
        self.arch = arch
        self.net = Net(arch, max_batch=int(model_info.get("max_batch", 512)), device=self.device)
        rng = np.random.default_rng(self._init_seed) if self._init_seed is not None else np.random.default_rng()
        glorot_uniform_(self.net, rng)
        mode = capi.CLIP_PER_TENSOR if self.clipnorm else capi.CLIP_NONE
        # keras Adam: epsilon = K.epsilon() = 1e-7
        self.opt = Adam(self.net, self.learning_rate, eps=1e-7, clip_mode=mode, clip=float(self.clipnorm or 0.0))
        self.q_name = arch["outputs"][0]   # the dueling combine layer when model_config has dueling: True
        self._obs_dt = torch.uint8 if arch["input_dtype"] == "uint8" else torch.float32
        self._np_dt = np.uint8 if arch["input_dtype"] == "uint8" else np.float32
        self._bufs = {}
        return self.net

    def _buffers(self, n):
        b = self._bufs.get(n)
        if b is None:
            dev = self.device
            b = dict(obs=torch.empty((n,) + tuple(self.state_dim), dtype=self._obs_dt, device=dev),
                     y=torch.empty(n, self.action_dim, dtype=torch.float32, device=dev),
                     loss=torch.zeros(1, dtype=torch.float32, device=dev))
            self._bufs[n] = b
        return b

    def forward_device(self, obs, n):
        self.net.ensure_batch(n)
        self.net.forward(obs, n)
        return self.net.tensor(self.q_name)[:n]

    def predict(self, state):
        """dqn_cnn.py:73-83: Q values [B, A]."""
        state = np.ascontiguousarray(state, self._np_dt)
        n = state.shape[0]
        b = self._buffers(n)
        b["obs"].copy_(torch.from_numpy(state), non_blocking=True)
        return self.forward_device(b["obs"], n).cpu().numpy()

    def train(self, state, label):
        """XTModel.train = keras train_on_batch(state, y) with loss 'mse' (xt/model/model.py:77-82)."""
        state = np.ascontiguousarray(state, self._np_dt)
        n = state.shape[0]
        b = self._buffers(n)
        b["obs"].copy_(torch.from_numpy(state), non_blocking=True)
        b["y"].copy_(torch.from_numpy(np.ascontiguousarray(label, np.float32)))
        net = self.net
        q = self.forward_device(b["obs"], n)
        b["loss"].zero_()
        check(net.lib.xtb_mse_loss_grad(_ptr(q), _ptr(b["y"]), n, self.action_dim, 1.0 / (n * self.action_dim),
                                        _ptr(net.tensor_grad(self.q_name)), _ptr(b["loss"]), stream_ptr()))
        net.backward(b["obs"], n, [self.q_name])
        self.opt.step()
        return float(b["loss"].cpu()[0])

    def train_td_device(self, target_model, obs, action, reward, next_obs, done, n, gamma, loss_buf, double_dqn=False,
                        idx=None, disc=None, huber_delta=0.0):
        """Fused DQN.train (xt/algorithm/dqn/dqn.py:61-97) on device-resident transitions: target forward,
        (double-DQN online forward on s'), online forward on s, TD target + loss gradient, backward, Adam -- one native
        call replayed as a CUDA graph.  `idx` (int32 device tensor): the step uses rows idx[0..n) of the given buffers
        (a replay ring) without copying them; `disc`: per-row n-step bootstrap discount; huber_delta > 0: Huber loss."""
        net = self.net
        net.ensure_batch(n)
        target_model.net.ensure_batch(n)
        key = ("td", n)
        sc = self._bufs.get(key)
        if sc is None:
            sc = dict(qn_t=torch.empty(n, self.action_dim, dtype=torch.float32, device=self.device),
                      qn_o=torch.empty(n, self.action_dim, dtype=torch.float32, device=self.device))
            self._bufs[key] = sc
        loss_buf.zero_()
        check(net.lib.xtb_dqn_train(net.handle, target_model.net.handle, self.opt.handle, _ptr(obs), _ptr(next_obs), _ptr(idx),
                                    _ptr(action), _ptr(reward), _ptr(done), _ptr(disc), int(n), float(gamma), float(huber_delta),
                                    net.tid[self.q_name], _ptr(sc["qn_t"]), _ptr(sc["qn_o"]) if double_dqn else None,
                                    _ptr(loss_buf), 1 if self.use_graph else 0, stream_ptr()))
        return loss_buf


@Registers.model
class DqnCnn(_DqnBase):
    """conv32/64/64 -> 256 -> A (dueling: + 1, combined); Adam(lr, clipnorm=10) (dqn_cnn.py:45-61)."""
    clipnorm = 10.0

    def build_arch(self):
        return archs.dqn_cnn(self.state_dim, self.action_dim, dueling=self.dueling)


@Registers.model
class DqnMlp(_DqnBase):
    """Dense(HIDDEN_SIZE) x NUM_LAYERS -> A (dueling: + 1, combined); Adam(lr) (dqn_mlp.py:43-60)."""
    clipnorm = None

    def build_arch(self):
        return archs.dqn_mlp(self.state_dim, self.action_dim, HIDDEN_SIZE, NUM_LAYERS, dueling=self.dueling)
