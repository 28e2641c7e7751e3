"""ImpalaCnnOpt on the CUDA engine (xt/model/impala/impala_cnn_opt.py:64-297)."""
import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, _ptr, stream_ptr
from ..registry import Registers, import_config
from . import archs
from .base import PolicyActor, XTModel

# xt/model/impala/default_config.py
LR = 0.0003
ENTROPY_LOSS = 0.01
GAMMA = 0.99


@Registers.model
class ImpalaCnnOpt(XTModel, PolicyActor):
    """IMPALA conv net with the V-trace loss evaluated inside the train step."""

    predict_head = True

    def __init__(self, model_info):
        model_config = model_info.get("model_config", dict())
        import_config(globals(), model_config)
        self.input_dtype = model_info.get("input_dtype", "float32")
        self.sta_mean = model_info.get("state_mean", 0.)
        self.sta_std = model_info.get("state_std", 255.)
        self.state_dim = model_info["state_dim"]
        self.action_dim = model_info["action_dim"]
        self.lr_schedule = model_config.get("lr_schedule", None)
        self.opt_type = model_config.get("opt_type", "adam")
        self.lr = LR
        self.grad_norm_clip = model_config.get("grad_norm_clip", 40.0)
        self.sample_batch_steps = model_config.get("sample_batch_step", 50)
        if self.opt_type not in ("adam", "rmsprop"):
            raise KeyError("invalid opt_type: {}".format(self.opt_type))          # impala_cnn_opt.py:207-208
        if self.lr_schedule and len(self.lr_schedule) != 2:
            raise ValueError("lr_schedule invalid: {}".format(self.lr_schedule))  # impala_cnn_opt.py:237-240 (logging.fatal)
        if self.input_dtype not in ("uint8",) or abs(self.sta_mean) >= 1e-4:
            # state_transform (model_utils.py:192-201): uint8 with mean~0 => x/std
            raise NotImplementedError("ImpalaCnnOpt: only uint8 observations with state_mean 0 are supported")
        super().__init__(model_info)

    def create_model(self, model_info):
        arch = archs.impala_cnn(self.state_dim, self.action_dim)
        arch["scale"] = 1.0 / float(self.sta_std)
        self.arch = arch
        self.net = self.seeded_net(arch, int(model_info.get("max_batch", 512)))
        # baseline head: custom_norm_initializer(0.01) (model_utils.py:204-211, impala_cnn_opt.py:146)
        name = "explore_agent/dense/kernel"
        shape = self.net.ptable[name][1]
        o = self._init_rng.standard_normal(shape).astype(np.float32)
        o *= 0.01 / np.sqrt(np.square(o).sum(axis=0, keepdims=True))
        self.net.view(name).copy_(torch.from_numpy(o))
        self.net.params_changed()
        self.opt = Adam(self.net, self.lr, eps=1e-8, clip_mode=capi.CLIP_GLOBAL_NORM, clip=self.grad_norm_clip)
        if self.opt_type == "rmsprop":
            self.opt.use_rmsprop(decay=0.99, epsilon=0.1)          # impala_cnn_opt.py:205-206 (the schedule is Adam-only there)
        self._global_step = 0
        self._bufs = {}
        self._init_sampling()
        self.logit_name, self.base_name = arch["outputs"]
        self.pi_t, self.v_t, self.ls_t = self.net.tid[self.logit_name], self.net.tid[self.base_name], 0
        return self.net

    def _buffers(self, n):
        b = self._bufs.get(n)
        if b is None:
            dev = self.device
            b = dict(obs=torch.empty((n,) + tuple(self.state_dim), dtype=torch.uint8, device=dev),
                     bp=torch.empty(n, self.action_dim, dtype=torch.float32, device=dev),
                     action=torch.empty(n, dtype=torch.int32, device=dev),
                     done=torch.empty(n, dtype=torch.uint8, device=dev),
                     reward=torch.empty(n, dtype=torch.float32, device=dev),
                     logp=torch.empty(n, dtype=torch.float32, device=dev),
                     loss=torch.zeros(1, dtype=torch.float32, device=dev))
            self._bufs[n] = b
        return b

    def train_device(self, obs, bp_logits, actions, dones, rewards, n, loss_buf):
        """One V-trace SGD step on device-resident tensors ([n] env-major, n = k*sample_batch_step)."""
        net = self.net
        s = int(self.sample_batch_steps)
        if n % s != 0 or n < s:
            raise ValueError("batch of %d samples is not a whole number of %d-step trajectories" % (n, s))
        net.ensure_batch(n)
        loss_buf.zero_()
        if self.lr_schedule and self.opt_type == "adam":
            self.opt.set_lr(self.scheduled_lr(self._global_step))
        self._global_step += 1
        # forward, in-graph V-trace + losses, backward, clip + Adam: one native call, replayed as a CUDA graph
        check(net.lib.xtb_impala_train(net.handle, self.opt.handle, _ptr(obs), None, _ptr(bp_logits), _ptr(actions), _ptr(dones),
                                       _ptr(rewards), int(n), s, float(GAMMA), net.tid[self.logit_name], net.tid[self.base_name],
                                       _ptr(loss_buf), 1 if self.use_graph else 0, stream_ptr()))
        return loss_buf

    def scheduled_lr(self, global_step, decay_step=20000.0):
        """impala_cnn_opt.py:234-249: tf.train.linear_cosine_decay(lr_schedule[0][1], global_step, 20000,
        beta=lr_schedule[1][1] / 20000) with the TF defaults num_periods=0.5, alpha=0:
        lr * ((alpha + (D - s) / D) * 0.5 * (1 + cos(pi * 2 * num_periods * s / D)) + beta), s = min(global_step, D)."""
        import math
        base, beta = float(self.lr_schedule[0][1]), float(self.lr_schedule[1][1]) / float(decay_step)
        s = min(float(global_step), float(decay_step))
        linear = (decay_step - s) / decay_step
        cosine = 0.5 * (1.0 + math.cos(math.pi * 2.0 * 0.5 * s / decay_step))
        return base * (linear * cosine + beta)

    def train(self, state, label):
        """impala_cnn_opt.py:251-265: train(state, [bp_logic_outs, actions, dones, rewards]) -> loss."""
        bp_logic_outs, actions, dones, rewards = label
        n = len(state)
        b = self._buffers(n)
        b["obs"].copy_(torch.from_numpy(np.ascontiguousarray(state, np.uint8)), non_blocking=True)
        b["bp"].copy_(torch.from_numpy(np.ascontiguousarray(bp_logic_outs, np.float32)))
        b["action"].copy_(torch.from_numpy(np.ascontiguousarray(actions, np.int32).reshape(-1)))
        b["done"].copy_(torch.from_numpy(np.ascontiguousarray(dones, np.bool_).reshape(-1).view(np.uint8)))
        b["reward"].copy_(torch.from_numpy(np.ascontiguousarray(rewards, np.float32).reshape(-1)))
        loss = self.train_device(b["obs"], b["bp"], b["action"], b["done"], b["reward"], n, b["loss"])
        return float(loss.cpu()[0])

    def predict(self, state, uniforms=None):
        """impala_cnn_opt.py:267-277: [logits [B,A], baseline [B], action [B]]."""
        state = np.ascontiguousarray(state, np.uint8)
        n = state.shape[0]
        net = self.net
        if uniforms is None and n <= net.max_batch:
            io = self._predict_host(state)
            out = io["pin_out_np"]
            return [io["pin_head"].numpy().copy(), out[2].copy(), out[0].view(np.int32).copy()]
        b = self._buffers(n)
        net.ensure_batch(n)
        b["obs"].copy_(torch.from_numpy(state), non_blocking=True)
        net.forward(b["obs"], n)
        u = None
        if uniforms is not None:
            u = torch.from_numpy(np.ascontiguousarray(uniforms, np.float32)).to(self.device)
        self._draw(n, b["action"], b["logp"], u)
        logits = net.tensor(self.logit_name)[:n].cpu().numpy()
        base = net.tensor(self.base_name)[:n, 0].cpu().numpy()
        return [logits, base, b["action"].cpu().numpy()]
