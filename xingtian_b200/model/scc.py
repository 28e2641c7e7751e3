"""SCCModel on the CUDA engine (xt/model/scc/scc_tf.py): Shapley counterfactual credits (KDD 2021).

The agent network and its explore step are QMixModel's (xt/model/qmix), and so is their device code.  What SCC adds is
the learner: a critic over every agent's (raw observation, one-hot action), per agent group ("multi-channel") or over
the whole row, trained by Adam on a TD loss, and counterfactual credits that the agents regress their chosen Q onto with
plain RMSProp.  A weight set is one flat buffer [fc1 | GRU | fc2 | critic nets | head]; the train graph has no target
agent, so only the critic part of the target set is used.  The training step (xtb_scc_train), the one-step inference
(xtb_scc_infer) and the critic (xtb_scc_critic) run in libxtb200."""
import ctypes as C
import random
from types import SimpleNamespace

import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, Net, _ptr, stage_h2d, stream_ptr
from ..registry import Registers
from .qmix import QMixModel, _align
from .base import XTModel

# agent_group_dict of scc_tf.py:56: agents per group of the multi-channel critic, by SMAC map; any other map is one group
AGENT_GROUPS = {"2s3z": [2, 3], "3s5z": [3, 5], "3s5z_vs_3s6z": [3, 5], "1c3s5z": [1, 3, 5], "MMM2": [1, 2, 7]}


@Registers.model
class SCCModel(QMixModel):
    """SCCModel (scc_tf.py:39-707).  model_info["scene"] = "explore" builds the acting network only, "train" also the
    eval agent and both critics.  The agent, weights, saving and the explore step are QMixModel's."""

    _native = "xtb_scc"

    def __init__(self, model_info):
        model_config = self._agent_config(model_info)
        map_name = model_config["map_name"]
        self.agent_group = list(AGENT_GROUPS[map_name]) if map_name in AGENT_GROUPS else [model_config["n_agents"]]
        self.c_lr = model_config.get("c_lr", 0.0005)
        self.a_lr = model_config.get("a_lr", 0.0005)
        self.mixer_grad_norm_clip = model_config.get("mixer_grad_norm_clip", 10)
        self.actor_grad_norm_clip = model_config.get("actor_grad_norm_clip", 10)
        self.use_double_q = model_config.get("use_double_q", True)
        self.o_shape = self.obs_shape - self.n_actions - self.n_agents
        if self.g_type == "train":
            # read when the train graph is built (scc_tf.py:280-313, 379-380)
            if not self.use_double_q:
                raise RuntimeError("double q is needed")
            self.dense_unit_number = int(model_config["dense_unit_number"])
            self.multi_channel = bool(model_config["enable_critic_multi_channel"])
            self.channel_merge = model_config["channel_merge"] if self.multi_channel else None
            if self.multi_channel and self.channel_merge not in ("concat", "add"):
                raise RuntimeError("Channel merge method is not correct")
            self.mc_sample_times = int(model_config.get("mc_sample_times", 1)) if self.n_agents > 2 else 1
        XTModel.__init__(self, model_info)

    # ---- construction ---------------------------------------------------------------------------------------------
    def create_model(self, model_info):
        A, n = self.n_actions, self.n_agents
        train = self.g_type == "train"
        B, L = self._agent_nets(train)
        self.critics = []
        end = self.agent_size
        if train:
            U, D, BL = self.dense_unit_number, self.o_shape + A, B * L
            if self.o_shape < 0:
                raise ValueError("obs_shape {} is narrower than n_actions + n_agents".format(self.obs_shape))
            # multi-channel: one net per group over its agents' (obs, action) slices; else one net over the whole row
            groups = self.agent_group if self.multi_channel else [None]
            self.n_variants = 0 if self.multi_channel else (n if n <= 2 else 2 * n * self.mc_sample_times)
            for j, g in enumerate(groups):
                width, max_rows = (D, BL * g) if g is not None else (n * D, BL * max(1, self.n_variants))
                arch = dict(input_dtype="float32", state_dim=(width,), scale=1.0, layers=[
                    ("dense", "dense", "obs", dict(n=U, act="relu")), ("dense_1", "dense", "dense", dict(n=U, act="relu"))])
                self.critics.append(Net(arch, max_batch=max_rows, device=self.device))
            self.o_mix = _align(end)
            o = self.o_mix
            for j, net in enumerate(self.critics):
                scope = "channel_%d/" % j if self.multi_channel else "critic/"
                for name, (po, shape) in net.ptable.items():
                    self.mixer_vars[scope + name] = (o + po, shape)
                net.o = o
                o = _align(o + net.n_params)
            self.head_off = o
            K = n * U if self.multi_channel and self.channel_merge == "concat" else U
            self.mixer_vars["v/kernel"] = (o, (K, 1))
            self.mixer_vars["v/bias"] = (o + K, (1,))
            end = o + K + 1
        self.n_params = end
        # the sub-graphs initialised as scc_tf.py:180-182, 321-391 builds them: the train graph has no target agent
        self._weight_sets([(c, c.o) for c in self.critics], target_agent=False)
        dev = self.device
        self.opt = self.critic_opt = None
        desc = capi.SccDesc()
        desc.batch, desc.episode_limit, desc.n_agents, desc.gamma, desc.gru_off = B, L, n, float(self.gamma), self.gru_off
        desc.act_envs = self.act_envs
        if train:
            clip = self.actor_grad_norm_clip > 0      # scc_tf.py:421: both clips, or neither
            mode = capi.CLIP_PER_TENSOR if clip else capi.CLIP_NONE
            astarts = [o for o, _ in self.agent_vars.values()] + [self.agent_size]
            aflat = SimpleNamespace(params=self.params[:self.agent_size], n_params=self.agent_size, device=dev,
                                    segment_offsets=lambda: astarts)
            cstarts = [o - self.o_mix for o, _ in self.mixer_vars.values()] + [self.n_params - self.o_mix]
            cflat = SimpleNamespace(params=self.params[self.o_mix:], n_params=self.n_params - self.o_mix, device=dev,
                                    segment_offsets=lambda: cstarts)
            # tf.train.AdamOptimizer(c_lr) for the critic, tf.train.RMSPropOptimizer(a_lr) (decay 0.9, epsilon 1e-10,
            # uncentred) for the agent, each variable's gradient clip_by_norm'ed
            self.critic_opt = Adam(cflat, self.c_lr, eps=1e-8, clip_mode=mode, clip=float(self.mixer_grad_norm_clip) if clip else 0.0)
            self.opt = Adam(aflat, self.a_lr, clip_mode=mode, clip=float(self.actor_grad_norm_clip) if clip else 0.0)
            self.opt.use_rmsprop(decay=0.9, epsilon=1e-10, centered=False)
            desc.head_off = self.head_off
            desc.mc_sample_times = self.mc_sample_times
            if self.multi_channel:
                desc.n_groups = len(self.agent_group)
                for j, g in enumerate(self.agent_group[:8]):
                    desc.group[j] = int(g)
                desc.channel_merge = 0 if self.channel_merge == "concat" else 1
        else:
            # the explore scene: the agent only, under a one-net critic that is never run
            desc.head_off = 0
        self.handle = C.c_void_p()
        if train:
            nets = (C.c_void_p * len(self.critics))(*[c.handle.value for c in self.critics])
            with torch.cuda.device(dev):
                check(capi.lib().xtb_scc_create(self.fc1.handle, self.fc2.handle, nets, C.byref(desc), C.byref(self.handle)))
        else:
            self._explore_handle()
        self._acting_state()
        self.mixer_loss = self.actor_loss = None
        return self.fc1

    def _explore_handle(self):
        """The explore scene has no critic: a minimal one-group critic (one unit, one-action slices) is created beside
        the agent so that xtb_scc_infer has an object to run on; it is never trained or evaluated."""
        n, A = self.n_agents, self.n_actions
        arch = dict(input_dtype="float32", state_dim=(A,), scale=1.0, layers=[
            ("dense", "dense", "obs", dict(n=1, act="relu")), ("dense_1", "dense", "dense", dict(n=1, act="relu"))])
        stub = Net(arch, max_batch=n, device=self.device)
        o = _align(self.agent_size)
        head = _align(o + stub.n_params)
        self._stub_params = torch.zeros(head + 1 + n + 1, dtype=torch.float32, device=self.device)
        self._stub_grads = torch.zeros_like(self._stub_params)
        fc = [(self.fc1, 0), (self.fc2, self.agent_vars["dense_1/kernel"][0]), (stub, o)]
        # the agent nets stay bound to the explore-scene eval set; the stub critic sits behind it in the same buffer
        self._stub_params[:self.agent_size].copy_(self.params[:self.agent_size])
        for net, off in fc:
            net.bind_to(self._stub_params[off:off + net.n_params], self._stub_grads[off:off + net.n_params])
            net.params_changed()
        self.params, self.grads, self._stub = self._stub_params, self._stub_grads, stub
        desc = capi.SccDesc()
        desc.batch, desc.episode_limit, desc.n_agents, desc.gru_off, desc.head_off = 1, 1, n, self.gru_off, head
        desc.n_groups, desc.group[0], desc.channel_merge, desc.mc_sample_times = 1, n, 1, 1
        desc.act_envs = self.act_envs
        nets = (C.c_void_p * 1)(stub.handle.value)
        with torch.cuda.device(self.device):
            check(capi.lib().xtb_scc_create(self.fc1.handle, self.fc2.handle, nets, C.byref(desc), C.byref(self.handle)))

    # ---- weights ----------------------------------------------------------------------------------------------------
    def assign_targets(self):
        """eval mixer -> target mixer (scc_tf.py:450-457); the agent has no target."""
        if self.mixer_vars:
            self.target[self.o_mix:].copy_(self.params[self.o_mix:])

    # ---- critic -----------------------------------------------------------------------------------------------------
    def _require_train(self, what):
        if self.opt is None:
            raise RuntimeError("SCCModel.{} needs the train scene".format(what))

    def get_mixer_output(self, critic_state):
        """V of the eval critic (scc_tf.py:500-503) on critic states [..., n_agents (o + n_actions)] -> [..., 1]."""
        self._require_train("get_mixer_output")
        s = np.asarray(critic_state, dtype=np.float32)
        width = self.n_agents * (self.o_shape + self.n_actions)
        if s.shape[-1] != width:
            raise ValueError("critic states are {} wide, not {}".format(s.shape[-1], width))
        flat = s.reshape(-1, width)
        cap = self._B * self._L
        if getattr(self, "_crit_io", None) is None:
            self._crit_io = (torch.empty(cap, width, dtype=torch.float32, device=self.device),
                             torch.empty(cap, dtype=torch.float32, device=self.device))
        x, v = self._crit_io
        out = np.empty(flat.shape[0], np.float32)
        for r0 in range(0, flat.shape[0], cap):
            rows = min(cap, flat.shape[0] - r0)
            stage_h2d(x[:rows], flat[r0:r0 + rows], np.float32)
            check(capi.lib().xtb_scc_critic(self.handle, _ptr(x), rows, _ptr(v), 1 if self.use_graph else 0, stream_ptr()))
            out[r0:r0 + rows] = v[:rows].cpu().numpy()
        return out.reshape(s.shape[:-1] + (1,))

    def get_ex_according_to_mcshap_mask(self, ep_critic_state, n_agents, n_obs, n_actions):
        """Monte-Carlo Shapley credits (scc_tf.py:658-690), the critic evaluated on the device; draws from Python's
        global `random` as the reference does."""
        ep_critic_state = np.array(ep_critic_state)
        mc_times = self.model_config["mc_sample_times"]
        shapley_agents = []
        for i in range(n_agents):
            shapley_list = []
            for _ in range(mc_times):
                agents_no = [x for x in range(n_agents)]
                agents_no.remove(i)
                sample_num = random.randint(1, n_agents - 1)
                agents_no = random.sample(agents_no, sample_num)
                mask_with_i = np.ones_like(ep_critic_state)
                mask_without_i = np.ones_like(ep_critic_state)
                for ag in agents_no:
                    mask_with_i[:, :, ag * (n_obs + n_actions) + n_obs:(ag + 1) * (n_obs + n_actions)] = 0
                    mask_without_i[:, :, ag * (n_obs + n_actions) + n_obs:(ag + 1) * (n_obs + n_actions)] = 0
                mask_without_i[:, :, i * (n_obs + n_actions) + n_obs:(i + 1) * (n_obs + n_actions)] = 0
                v_with_i = self.get_mixer_output(mask_with_i * ep_critic_state)
                v_without_i = self.get_mixer_output(mask_without_i * ep_critic_state)
                shapley_list.append(v_with_i - v_without_i)
            shapley_agents.append(np.mean(np.stack(shapley_list, 0), 0))
        return np.stack(shapley_agents, 2)

    def get_ex_according_to_mask(self, ep_critic_state, n_agents, n_obs, n_actions):
        """Counterfactual credits (scc_tf.py:693-707): V minus V with agent i's whole slice zeroed."""
        ep_critic_state = np.array(ep_critic_state)
        credit_agents = []
        for i in range(n_agents):
            mask_i = np.ones_like(ep_critic_state)
            mask_i[:, :, i * (n_obs + n_actions):(i + 1) * (n_obs + n_actions)] = 0
            credit_agents.append(self.get_mixer_output(ep_critic_state) - self.get_mixer_output(mask_i * ep_critic_state))
        return np.stack(credit_agents, 2)

    # ---- training ---------------------------------------------------------------------------------------------------
    def draw_subsets(self):
        """The reference's Monte-Carlo subset draws for one train call (scc_tf.py:662-668), in its order from Python's
        global `random`: [n_agents, mc_sample_times] agent bitmasks.  Made whenever n_agents > 2, whichever critic, so
        that the stream advances as in the reference."""
        n, mc = self.n_agents, self.model_config["mc_sample_times"]
        out = np.zeros((n, mc), np.uint32)
        for i in range(n):
            for j in range(mc):
                agents_no = [x for x in range(n)]
                agents_no.remove(i)
                sample_num = random.randint(1, n - 1)
                for a in random.sample(agents_no, sample_num):
                    out[i, j] |= np.uint32(1 << a)
        return out

    def _train_buffers(self):
        if self._bufs is None:
            B, L, n, dev = self._B, self._L, self.n_agents, self.device
            f32 = dict(dtype=torch.float32, device=dev)
            self._bufs = dict(obs=torch.empty(B, L + 1, n, self.obs_shape, **f32),
                              raw_obs=torch.empty(B, L + 1, n, max(self.o_shape, 1), **f32),
                              seq_len=torch.empty(B * n, dtype=torch.int32, device=dev),
                              actions=torch.empty(B, L, n, dtype=torch.int32, device=dev),
                              reward=torch.empty(B, L, **f32), terminated=torch.empty(B, L, **f32), mask=torch.empty(B, L, **f32),
                              subsets=torch.zeros(n, max(1, self.mc_sample_times), dtype=torch.int32, device=dev),
                              loss=torch.zeros(2, **f32))
        return self._bufs

    def train(self, batch_trajectories, obs, train_obs_len, avail_actions, actions, cur_stats, target_stats, rewards, terminated,
              mask):
        """scc_tf.py:505-564: the critic's Adam step and the agents' RMSProp step on one batch -> actor loss + mixer loss
        (both kept: self.mixer_loss, self.actor_loss).  avail_actions and the states are not read by the train graph."""
        self._require_train("train")
        B, L, n = self._B, self._L, self.n_agents
        raw = np.asarray(obs)
        if raw.shape[-1] != self.o_shape:
            raise ValueError("obs is {} wide, not obs_shape - n_actions - n_agents = {}".format(raw.shape[-1], self.o_shape))
        seq_len, act = self._agent_batch(train_obs_len, actions)
        subsets = self.draw_subsets() if n > 2 else None
        b = self._train_buffers()
        stage_h2d(b["obs"], batch_trajectories, np.float32)
        if self.o_shape:
            # with no raw observation columns the critic states are the one-hot actions alone: nothing reads raw_obs
            stage_h2d(b["raw_obs"], raw.reshape(B, L + 1, n, self.o_shape), np.float32)
        stage_h2d(b["seq_len"], seq_len, np.int32)
        stage_h2d(b["actions"], act, np.int32)
        stage_h2d(b["reward"], rewards, np.float32)
        stage_h2d(b["terminated"], terminated, np.float32)
        stage_h2d(b["mask"], mask, np.float32)
        if subsets is not None:
            stage_h2d(b["subsets"], subsets.view(np.int32)[:, :b["subsets"].shape[1]], np.int32)
        self.train_device(b)
        mixer, actor = b["loss"].cpu().numpy()
        self.mixer_loss, self.actor_loss = float(mixer), float(actor)
        return float(actor + mixer)

    def train_replay(self, replay, ids):
        """SCCAlg.train's step on the episodes `ids` of a DeviceEpisodeReplay (xtb_scc_replay_train): as
        QMixModel.train_replay, with the raw obs gathered from the ring and the Monte-Carlo subsets drawn and uploaded
        as train() does -> (actor + mixer loss, max_t_filled)."""
        self._require_train("train_replay")
        subsets = self.draw_subsets() if self.n_agents > 2 else None
        b = self._train_buffers()
        if subsets is not None:
            stage_h2d(b["subsets"], subsets.view(np.int32)[:, :b["subsets"].shape[1]], np.int32)
        out = self._replay_out(2)
        bt = capi.SccBatch()
        for k in ("obs", "raw_obs", "seq_len", "actions", "reward", "terminated", "mask", "subsets"):
            setattr(bt, k, b[k].data_ptr())
        ids = np.ascontiguousarray(ids, np.int32)
        check(capi.lib().xtb_scc_replay_train(replay.handle, self.handle, self.critic_opt.handle, self.opt.handle, _ptr(self.target),
                                              len(ids), ids.ctypes.data, C.byref(bt), _ptr(out[:2]), _ptr(out[2:]),
                                              1 if self.use_graph else 0, stream_ptr()))
        host = out.cpu().numpy()
        mixer, actor = host[:2]
        self.mixer_loss, self.actor_loss = float(mixer), float(actor)
        return float(actor + mixer), int(host[2:].view(np.int32)[0])

    def train_device(self, b):
        """xtb_scc_train on the device tensors of _train_buffers(); [mixer loss, actor loss] land in b["loss"]."""
        bt = capi.SccBatch()
        for k in ("obs", "raw_obs", "seq_len", "actions", "reward", "terminated", "mask", "subsets"):
            setattr(bt, k, b[k].data_ptr())
        check(capi.lib().xtb_scc_train(self.handle, self.critic_opt.handle, self.opt.handle, _ptr(self.target), C.byref(bt),
                                       _ptr(b["loss"]), 1 if self.use_graph else 0, stream_ptr()))
