"""ImpalaMlp / ImpalaCnn on the CUDA engine (xt/model/impala/impala_mlp.py:39-93, impala_cnn.py:44-108): the Keras
models IMPALA trains.  The `output_actions` softmax, the hand-written `impala_loss` + 0.5 mse and the Keras fit epoch run
on the device; the two concrete models live in modules of their own (impala_mlp.py, impala_cnn.py) so that
import_config writes each one's own module globals, as in the reference."""
import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, Net, _ptr, stage_h2d, stream_ptr
from ..registry import import_config
from .base import XTModel, glorot_uniform_

FIT_BATCH = 128   # model.fit(batch_size=128) (impala_mlp.py:64-71, impala_cnn.py:79-86)


def fit_order(n):
    """training_arrays.fit_loop with shuffle=True (TF-1.15): one np.random.shuffle(np.arange(n)) per fit call; the
    minibatches are its consecutive FIT_BATCH-row pieces, the last one ragged."""
    order = np.arange(n)
    np.random.shuffle(order)
    return order


class ImpalaKerasModel(XTModel):
    """Shared body of ImpalaMlp / ImpalaCnn.  Sub-classes set `config` (their module globals), `clipnorm`, `decay` and
    build_arch()."""
    config = None
    clipnorm = None
    decay = 0.0

    def __init__(self, model_info):
        model_config = model_info.get("model_config", None) or {}
        import_config(self.config, model_config)
        self.state_dim = model_info["state_dim"]
        self.action_dim = model_info["action_dim"]
        self.learning_rate = self.config["LR"]
        self.ent_coef = self.config["ENTROPY_LOSS"]
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
        if self.decay:
            self.opt.set_decay(self.decay)
        self.logit_name, self.value_name = arch["outputs"]
        self._obs_dt = torch.uint8 if arch["input_dtype"] == "uint8" else torch.float32
        self._np_dt = np.uint8 if arch["input_dtype"] == "uint8" else np.float32
        self._bufs = {}
        return self.net

    def _buffers(self, n):
        b = self._bufs.get(n)
        if b is None:
            dev = self.device
            b = dict(obs=torch.empty((n,) + tuple(self.state_dim), dtype=self._obs_dt, device=dev),
                     order=torch.empty(n, dtype=torch.int32, device=dev),
                     y=torch.empty(n, self.action_dim, dtype=torch.float32, device=dev),
                     adv=torch.empty(n, dtype=torch.float32, device=dev),
                     tv=torch.empty(n, dtype=torch.float32, device=dev),
                     probs=torch.empty(n, self.action_dim, dtype=torch.float32, device=dev),
                     loss=torch.zeros(1, dtype=torch.float32, device=dev))
            self._bufs[n] = b
        return b

    def predict_device(self, obs, n):
        """probs [n, A] (softmax of output_actions) and value [n, 1] of device observations, as device tensors."""
        net = self.net
        net.ensure_batch(n)
        net.forward(obs, n)
        probs = self._buffers(n)["probs"]
        check(net.lib.xtb_softmax(_ptr(net.tensor(self.logit_name)), n, self.action_dim, _ptr(probs), stream_ptr()))
        return probs, net.tensor(self.value_name)[:n]

    def predict(self, state):
        """impala_mlp.py:73-78: predict([obs, adv]) -> [probs [B, A], value [B, 1]] (adv is not used)."""
        obs = np.ascontiguousarray(state[0], self._np_dt)
        n = obs.shape[0]
        b = self._buffers(n)
        stage_h2d(b["obs"], obs, self._np_dt)
        probs, value = self.predict_device(b["obs"], n)
        return [probs.cpu().numpy(), value.cpu().numpy()]

    def fit_device(self, obs, order, action_mat, adv, target_v, n, loss_buf):
        """One Keras fit epoch over n device rows, minibatch k = rows order[k*128 ...]: forward, loss, backward and Adam
        per minibatch, one native call replayed as a CUDA graph.  loss_buf[0] = the epoch loss."""
        net = self.net
        net.ensure_batch(min(n, FIT_BATCH))
        check(net.lib.xtb_impala_keras_fit(net.handle, self.opt.handle, _ptr(obs), _ptr(order), _ptr(action_mat), _ptr(adv),
                                           _ptr(target_v), int(n), FIT_BATCH, net.tid[self.logit_name], net.tid[self.value_name],
                                           float(self.ent_coef), _ptr(loss_buf), 1 if self.use_graph else 0, stream_ptr()))
        return loss_buf

    def train(self, state, label):
        """impala_mlp.py:64-71: model.fit(x=[obs, adv], y=[action_matrix, target_value], batch_size=128) -> epoch loss."""
        obs = np.ascontiguousarray(state[0], self._np_dt)
        n = obs.shape[0]
        b = self._buffers(n)
        stage_h2d(b["obs"], obs, self._np_dt)
        stage_h2d(b["adv"], np.asarray(state[1]).reshape(-1), np.float32)
        stage_h2d(b["y"], np.asarray(label[0]), np.float32)
        stage_h2d(b["tv"], np.asarray(label[1]).reshape(-1), np.float32)
        stage_h2d(b["order"], fit_order(n), np.int32)
        return float(self.fit_device(b["obs"], b["order"], b["y"], b["adv"], b["tv"], n, b["loss"]).cpu()[0])
