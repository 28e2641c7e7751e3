"""PPO actor-critic on the CUDA engine: PPO / PpoCnn / PpoMlp (xt/model/ppo/*.py)."""
import ctypes as C

import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, DeviceStore, _ptr, stream_ptr
from ..registry import Registers, import_config
from . import archs
from .base import PolicyActor, XTModel

# xt/model/ppo/default_config.py:1-12
BATCH_SIZE = 200
CRITIC_LOSS_COEF = 1.0
ENTROPY_LOSS = 1e-3
LOSS_CLIPPING = 0.2
LR = 0.0003
NUM_SGD_ITER = 4
MAX_GRAD_NORM = 5.0
SUMMARY = False
VF_CLIP = 5.0
CNN_SHARE_LAYERS = True
MLP_SHARE_LAYERS = False

_SUPPORTED_ACT = tuple(capi.ACT)


def minibatch_order(nbatch, num_sgd_iter):
    """Index order of xt/model/ppo/ppo.py:114-121: `inds` is shuffled IN PLACE once per epoch with the
    global numpy RNG (so epoch e's order is a shuffle of epoch e-1's); returns int32 [num_sgd_iter, nbatch].
    Minibatch j of epoch e is row e, columns [j*BATCH_SIZE, (j+1)*BATCH_SIZE) -- the last one may be ragged."""
    inds = np.arange(nbatch)
    out = np.empty((num_sgd_iter, nbatch), np.int32)
    for e in range(num_sgd_iter):
        np.random.shuffle(inds)
        out[e] = inds
    return out


class DeviceRollout(DeviceStore):
    """Device-resident PPO rollout (grow-only, so CUDA-graph pointers stay valid).  With `action_dim` (a DiagGaussian
    actor) the behaviour actions are float32 [N, action_dim], else int32 [N]."""

    def __init__(self, state_dim, obs_dtype, device, action_dim=None):
        f32 = ((), torch.float32)
        super().__init__(device, obs=(tuple(state_dim), obs_dtype),
                         action=((), torch.int32) if action_dim is None else ((action_dim,), torch.float32),
                         old_logp=f32, adv=f32, old_v=f32, target_v=f32)

    def as_struct(self):
        return capi.PpoRollout(self.obs.data_ptr(), self.action.data_ptr(), self.old_logp.data_ptr(),
                               self.adv.data_ptr(), self.old_v.data_ptr(), self.target_v.data_ptr())


@Registers.model
class PPO(XTModel, PolicyActor):
    """Build PPO network (xt/model/ppo/ppo.py:37-132)."""

    def __init__(self, model_info):
        model_config = model_info.get("model_config")
        import_config(globals(), model_config)
        self.state_dim = model_info["state_dim"]
        self.action_dim = model_info["action_dim"]
        self.input_dtype = model_info.get("input_dtype", "float32")
        self.action_type = model_config.get("action_type", "Categorical")
        self._lr = model_config.get("LR", LR)
        self._batch_size = model_config.get("BATCH_SIZE", BATCH_SIZE)
        self.critic_loss_coef = model_config.get("CRITIC_LOSS_COEF", CRITIC_LOSS_COEF)
        self.ent_coef = model_config.get("ENTROPY_LOSS", ENTROPY_LOSS)
        self.clip_ratio = model_config.get("LOSS_CLIPPING", LOSS_CLIPPING)
        self._max_grad_norm = model_config.get("MAX_GRAD_NORM", MAX_GRAD_NORM)
        self.num_sgd_iter = model_config.get("NUM_SGD_ITER", NUM_SGD_ITER)
        self.verbose = model_config.get("SUMMARY", SUMMARY)
        self.vf_clip = model_config.get("VF_CLIP", VF_CLIP)
        if self.action_type not in ("Categorical", "DiagGaussian"):
            raise NotImplementedError(
                "action type: {} not match any implemented distributions.".format(self.action_type))
        # DiagGaussian (tf_dist.py:49-86, ppo.py:73-78): mean = pi_latent, log_std = the trainable pi_logstd (1, A)
        self.gaussian = self.action_type == "DiagGaussian"
        super().__init__(model_info)

    # -- graph construction ------------------------------------------------------------------
    def build_arch(self):
        raise NotImplementedError

    def create_model(self, model_info):
        arch = self.build_arch()
        self.arch = arch
        self.net = self.seeded_net(arch, max(int(self._batch_size), int(model_info.get("max_predict_batch", 1024))))
        self.opt = Adam(self.net, self._lr, eps=1e-8, clip_mode=capi.CLIP_GLOBAL_NORM, clip=self._max_grad_norm)
        self.hyper = capi.PpoHyper(self.clip_ratio, self.ent_coef, self.vf_clip, self.critic_loss_coef)
        self.rollout = DeviceRollout(self.state_dim, self._obs_dt, self.device, self.action_dim if self.gaussian else None)
        self._perm_dev = None
        self._perm_host = None
        self._loss_dev = None
        self._pred_bufs = {}
        self._obs_ring = None
        self._init_sampling()
        self.pi_t = self.net.tid["pi_latent"]
        self.v_t = self.net.tid["output_value"]
        self.ls_t = self.net.tid["pi_logstd"] if self.gaussian else 0
        return self.net

    # -- inference ---------------------------------------------------------------------------
    def _pred_buffers(self, batch):
        b = self._pred_bufs.get(batch)
        if b is None:
            dev = self.device
            action = torch.empty((batch, self.action_dim), dtype=torch.float32, device=dev) if self.gaussian else \
                torch.empty(batch, dtype=torch.int32, device=dev)
            b = dict(obs=torch.empty((batch,) + tuple(self.state_dim), dtype=self._obs_dt, device=dev), action=action,
                     logp=torch.empty(batch, dtype=torch.float32, device=dev))
            self._pred_bufs[batch] = b
        return b

    def predict_device(self, obs_dev, batch, uniforms=None, out_action=None, out_logp=None, idx=None, normals=None):
        """Batched inference on device-resident observations (row b = obs_dev[idx[b]] when idx is
        given); returns device views (action[B] i32, logp[B] f32, v[B,1] f32).  A DiagGaussian actor returns
        action [B, A] f32; `normals` [B, A] (device) then replaces the Philox draws, as `uniforms` does for Categorical."""
        net = self.net
        done = 0
        bufs = self._pred_buffers(batch) if out_action is None else None
        action = out_action if out_action is not None else bufs["action"]
        logp = out_logp if out_logp is not None else bufs["logp"]
        noise = normals if self.gaussian else uniforms
        vout = torch.empty(batch, 1, dtype=torch.float32, device=self.device) if batch > net.max_batch else None
        while done < batch:
            mb = min(net.max_batch, batch - done)
            if idx is None:
                net.forward(obs_dev[done:done + mb], mb)
            else:
                net.forward(obs_dev, mb, idx=idx[done:done + mb])
            self._draw(mb, action[done:done + mb], logp[done:done + mb], None if noise is None else noise[done:done + mb])
            if vout is not None:
                vout[done:done + mb].copy_(net.tensor("output_value")[:mb])
            done += mb
        v = vout if vout is not None else net.tensor("output_value")[:batch]
        return action[:batch], logp[:batch], v

    def predict(self, state, uniforms=None, normals=None):
        """xt/model/ppo/ppo.py:104-109: (action [B] int32, logp [B,1], v [B,1]); a DiagGaussian actor returns action
        [B, A] float32 (`normals` [B, A] then replaces the Philox draws)."""
        state = np.ascontiguousarray(state, dtype=self._np_dt)
        batch = state.shape[0]
        noise = normals if self.gaussian else uniforms
        if noise is not None or batch > self.net.max_batch:
            bufs = self._pred_buffers(batch)
            bufs["obs"].copy_(torch.from_numpy(state), non_blocking=True)
            if noise is not None:
                noise = torch.from_numpy(np.ascontiguousarray(noise, np.float32)).to(self.device)
            action, logp, v = self.predict_device(bufs["obs"], batch, None if self.gaussian else noise,
                                                  normals=noise if self.gaussian else None)
            return (action.cpu().numpy(), logp.cpu().numpy().reshape(batch, 1), v.cpu().numpy().reshape(batch, 1))
        io = self._predict_host(state)
        ring = self._obs_ring
        if ring is not None and batch == ring["E"]:
            # learner-side batched inference: the frames just uploaded ARE the rollout's cur_state -- keep them on the
            # device (time-major ring) so prepare_data can take them from here instead of a second H2D copy
            ring["obs"][ring["t"] % ring["T"]].copy_(io["obs"], non_blocking=True)
            ring["t"] += 1
        out = io["pin_out_np"]
        if self.gaussian:
            A = self.action_dim
            return (out[:A].reshape(batch, A).copy(), out[A].reshape(batch, 1).copy(), out[A + 1].reshape(batch, 1).copy())
        return (out[0].view(np.int32).copy(), out[1].reshape(batch, 1).copy(), out[2].reshape(batch, 1).copy())

    def keep_predict_obs(self, env_num, steps):
        """Enable the device observation ring [steps][env_num][...] filled by predict() (see Algorithm.prepare_data's
        `ring_rows` form).  Replaces the second upload of every frame (xt/framework/learner.py:382-437 data path)."""
        self._obs_ring = dict(E=int(env_num), T=int(steps), t=0,
                              obs=torch.empty((int(steps), int(env_num)) + tuple(self.state_dim), dtype=self._obs_dt, device=self.device))

    def heads_plan(self, infer):
        """(kpl, amax) of the fused-heads kernel that training (infer False) or rollout inference (infer True) launches
        for this policy's heads under the current fused-heads mode; (0, 0) when they run layer by layer."""
        kpl, amax = C.c_int(), C.c_int()
        check(self.net.lib.xtb_ppo_heads_plan(self.net.handle, self.pi_t, self.v_t, 1 if infer else 0, C.byref(kpl), C.byref(amax)))
        return kpl.value, amax.value

    # -- training ----------------------------------------------------------------------------
    def make_perm(self, nbatch):
        """Index order of xt/model/ppo/ppo.py:114-121: `inds` shuffled in place every epoch."""
        return minibatch_order(nbatch, self.num_sgd_iter)

    def train_device(self, nbatch, perm=None):
        """Run the minibatch-SGD loop on the device rollout (`self.rollout`, first nbatch rows)."""
        if perm is None:
            perm = self.make_perm(nbatch)
        perm = np.ascontiguousarray(perm, np.int32).reshape(-1)
        bs = int(self._batch_size)
        steps = self.num_sgd_iter * ((nbatch + bs - 1) // bs)
        if self._perm_dev is None or self._perm_dev.numel() < perm.size:
            self._perm_dev = torch.empty(perm.size, dtype=torch.int32, device=self.device)
            self._perm_host = torch.empty(perm.size, dtype=torch.int32).pin_memory()
        if self._loss_dev is None or self._loss_dev.numel() < steps:
            self._loss_dev = torch.zeros(steps, dtype=torch.float32, device=self.device)
        self._perm_host[:perm.size].copy_(torch.from_numpy(perm))
        self._perm_dev[:perm.size].copy_(self._perm_host[:perm.size], non_blocking=True)
        ro = self.rollout.as_struct()
        check(self.net.lib.xtb_ppo_train(self.net.handle, self.opt.handle, C.byref(ro), int(nbatch), bs, int(self.num_sgd_iter),
                                         _ptr(self._perm_dev), C.byref(self.hyper), self.pi_t, self.v_t, self.ls_t,
                                         _ptr(self._loss_dev), 1 if self.use_graph else 0, stream_ptr()))
        losses = self._loss_dev[:steps].cpu().numpy()
        self.last_losses = losses
        return float(np.mean(losses))

    def upload_rollout(self, state, label):
        nbatch = state[0].shape[0]
        ro = self.rollout
        ro.n = 0
        ro.reserve(nbatch)
        np_obs = np.ascontiguousarray(state[0], dtype=self._np_dt)
        ro.obs[:nbatch].copy_(torch.from_numpy(np_obs), non_blocking=True)
        if self.gaussian:
            act = np.ascontiguousarray(label[0], np.float32).reshape(nbatch, self.action_dim)
        else:
            act = np.ascontiguousarray(label[0], np.int32).reshape(-1)
        ro.action[:nbatch].copy_(torch.from_numpy(act))
        for key, arr in zip(("old_logp", "adv", "old_v", "target_v"), label[1:5]):
            getattr(ro, key)[:nbatch].copy_(torch.from_numpy(np.ascontiguousarray(arr, np.float32).reshape(-1)))
        ro.n = nbatch
        return nbatch

    def train(self, state, label):
        """xt/model/ppo/ppo.py:111-132.  state=[obs], label=[action, old_logp, adv, old_v, target_v]; action is float
        [N, A] for a DiagGaussian actor."""
        nbatch = self.upload_rollout(state, label)
        return self.train_device(nbatch)


@Registers.model
class PpoCnn(PPO):
    """xt/model/ppo/ppo_cnn.py:28-50."""

    def __init__(self, model_info):
        model_config = model_info.get("model_config")
        self.vf_share_layers = model_config.get("VF_SHARE_LAYERS", CNN_SHARE_LAYERS)
        self.hidden_sizes = model_config.get("hidden_sizes", [512])      # model_utils.py:110-117
        self.activation = model_config.get("activation", "relu")
        if self.activation not in _SUPPORTED_ACT:
            raise KeyError("activation {} not implemented.".format(self.activation))
        super().__init__(model_info)

    def build_arch(self):
        if self.input_dtype not in ("uint8", "float32"):
            raise ValueError("dtype: {} not supported automatically, please implement it yourself".format(self.input_dtype))
        arch = archs.ppo_cnn(self.state_dim, self.action_dim, self.hidden_sizes, self.activation, self.vf_share_layers,
                             diag_gaussian=self.gaussian)
        if self.input_dtype == "float32":
            arch["input_dtype"], arch["scale"] = "float32", 1.0
        return arch


@Registers.model
class PpoMlp(PPO):
    """xt/model/ppo/ppo_mlp.py:28-49."""

    def __init__(self, model_info):
        model_config = model_info.get("model_config")
        self.vf_share_layers = model_config.get("VF_SHARE_LAYERS", MLP_SHARE_LAYERS)
        self.hidden_sizes = model_config.get("hidden_sizes", [64, 64])   # model_utils.py:100-107
        self.activation = model_config.get("activation", "tanh")
        if self.activation not in _SUPPORTED_ACT:
            raise KeyError("activation {} not implemented.".format(self.activation))
        super().__init__(model_info)

    def build_arch(self):
        if self.input_dtype != "float32":
            raise ValueError("dtype: {} not supported automatically, please implement it yourself".format(self.input_dtype))
        return archs.ppo_mlp(self.state_dim, self.action_dim, self.hidden_sizes, self.activation, self.vf_share_layers,
                             diag_gaussian=self.gaussian)
