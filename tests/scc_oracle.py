"""Float64 restatement of SCCModel's train step (xt/model/scc/scc_tf.py:278-313, 398-448, 505-564, 657-707): the
critic states with the reference's shift, literal masked critic forwards for the credits (one per masked state, as the
reference evaluates them), both losses with autograd gradients, per-variable clip_by_norm, tf.train.AdamOptimizer for the
critic (oracle.xt_oracle.TFAdam) and uncentred tf.train.RMSPropOptimizer for the agent (TFRMSPropPlain).  The agent network is
QMIX's (tests/qmix_oracle.py).  The arithmetic type follows oracle.xt_oracle.precision."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import xt_oracle as orc
import qmix_oracle as qo

_t = qo._t


class TFRMSPropPlain(object):
    """tf.train.RMSPropOptimizer(lr, decay, epsilon) with its defaults centered=False and momentum 0, as documented for
    TF-1.15 (training_ops ApplyRMSProp): ms = rho ms + (1 - rho) g^2; theta -= lr g / sqrt(ms + eps); the `rms` slot is
    initialised to ONES.  (oracle.xt_oracle.TFRMSProp is the centred form.)"""

    def __init__(self, params, lr, decay=0.9, eps=1e-10):
        self.params, self.lr, self.rho, self.eps = params, lr, decay, eps
        self.ms = [torch.ones_like(p) for p in params]

    def step(self, grads):
        with torch.no_grad():
            for p, g, ms in zip(self.params, grads, self.ms):
                ms.mul_(self.rho).addcmul_(g, g, value=1 - self.rho)
                p.sub_(self.lr * g / (ms + self.eps).sqrt())


def critic_states(raw_obs, actions, n_actions):
    """scc_tf.py:535-546 in NumPy: s[b, t] = concat_a [obs[b, t, a], one_hot(actions[b, t, a])] (float64), t < L, then
    `next = s; next[:, :-1] = next[:, 1:]`.  `next` aliases s, so the returned states are the shifted ones:
    s'[b, t] = s[b, min(t + 1, L - 1)], which every critic evaluation and the credits read."""
    actions = np.asarray(actions)
    bs, n = actions.shape[0], actions.shape[2]
    one_hot = np.eye(n_actions)[actions.reshape(-1)]
    s = np.concatenate((np.asarray(raw_obs)[:, :-1], one_hot.reshape(bs, -1, n, n_actions)), -1).reshape(bs, -1, n * (raw_obs.shape[-1] + n_actions))
    nxt = s
    nxt[:, :-1] = nxt[:, 1:]
    return s


def _mlp(w, scope, x):
    h = torch.relu(x @ w[scope + "dense/kernel"] + w[scope + "dense/bias"])
    return torch.relu(h @ w[scope + "dense_1/kernel"] + w[scope + "dense_1/bias"])


def critic(w, s, cfg):
    """_build_mixer (scc_tf.py:278-313) on states [B, L, n D] -> V [B, L, 1]."""
    s = _t(s) if not torch.is_tensor(s) else s
    n = cfg["n_agents"]
    if not cfg["multi"]:
        return _mlp(w, "critic/", s) @ w["v/kernel"] + w["v/bias"]
    x = s.reshape(s.shape[0], s.shape[1], n, -1)
    hs, a = [], 0
    for j, g in enumerate(cfg["groups"]):
        for i in range(a, a + g):
            hs.append(_mlp(w, "channel_%d/" % j, x[:, :, i]))
        a += g
    hs = torch.cat(hs, 2) if cfg["merge"] == "concat" else sum(hs[1:], hs[0])
    return hs @ w["v/kernel"] + w["v/bias"]


def credits(w, s, cfg, subsets=None):
    """get_ex_according_to_mask (n <= 2) / get_ex_according_to_mcshap_mask (n > 2, the subsets as [n, mc] agent bitmasks
    in the reference's draw order) with literal masked states -> [B, L, n]."""
    n, D = cfg["n_agents"], s.shape[-1] // cfg["n_agents"]
    o = D - cfg["n_actions"]
    out = []
    with torch.no_grad():
        if n <= 2:
            v = critic(w, s, cfg)
            for i in range(n):
                m = np.ones_like(s)
                m[:, :, i * D:(i + 1) * D] = 0
                out.append(v - critic(w, m * s, cfg))
        else:
            for i in range(n):
                vals = []
                for j in range(subsets.shape[1]):
                    agents = [a for a in range(n) if (int(subsets[i, j]) >> a) & 1]
                    mw, mo = np.ones_like(s), np.ones_like(s)
                    for ag in agents:
                        mw[:, :, ag * D + o:(ag + 1) * D] = 0
                        mo[:, :, ag * D + o:(ag + 1) * D] = 0
                    mo[:, :, i * D + o:(i + 1) * D] = 0
                    vals.append(critic(w, mw * s, cfg) - critic(w, mo * s, cfg))
                out.append(torch.stack(vals, 0).mean(0))
    return torch.cat(out, -1)


def step_losses(wa, wc, wct, batch, cfg, subsets=None):
    """(mixer loss, actor loss, credits) of one train call; the credits come from wc before any update."""
    s = critic_states(batch["raw_obs"], batch["actions"], cfg["n_actions"])
    credit = credits(wc, s, cfg, subsets)
    v = critic(wc, s, cfg)[..., 0]
    with torch.no_grad():
        vt = critic(wct, s, cfg)[..., 0]
    mask = _t(batch["mask"])
    targets = _t(batch["reward"]) + cfg["gamma"] * (1 - _t(batch["terminated"])) * vt
    mixer = (((v - targets) * mask) ** 2).sum() / mask.sum()
    mac, _ = qo.agent_forward(wa, _t(batch["obs"]), batch["seq_len"])
    act = torch.as_tensor(np.asarray(batch["actions"]), dtype=torch.int64)
    chosen = torch.gather(mac[:, :-1], -1, act.unsqueeze(-1)).squeeze(-1)
    alive = mask.unsqueeze(-1).expand_as(chosen)
    actor = ((alive * chosen - alive * credit) ** 2).sum() / alive.sum()
    return mixer, actor, credit


class SccLearner(object):
    """Eval agent / eval and target critic weights {name: tensor} of the model's variable tables; Adam(c_lr) for the
    critic, uncentred RMSProp(a_lr, 0.9, 1e-10) for the agent, both clip_by_norm'ed per variable only when
    actor_grad_norm_clip > 0 (scc_tf.py:419-448)."""

    def __init__(self, agent_w, critic_w, target_w, cfg):
        self.wa = OrderedDict((k, _t(v).clone().requires_grad_(True)) for k, v in agent_w.items())
        self.wc = OrderedDict((k, _t(v).clone().requires_grad_(True)) for k, v in critic_w.items())
        self.wct = OrderedDict((k, _t(v)) for k, v in target_w.items())
        self.cfg = cfg
        self.copt = orc.TFAdam(list(self.wc.values()), cfg["c_lr"])
        self.aopt = TFRMSPropPlain(list(self.wa.values()), cfg["a_lr"], decay=0.9, eps=1e-10)

    def step(self, batch, subsets=None):
        mixer, actor, _ = step_losses(self.wa, self.wc, self.wct, batch, self.cfg, subsets)
        cg = torch.autograd.grad(mixer, list(self.wc.values()))
        ag = torch.autograd.grad(actor, list(self.wa.values()), allow_unused=True)
        ag = [torch.zeros_like(p) if g is None else g for p, g in zip(self.wa.values(), ag)]
        if self.cfg["actor_clip"] > 0:
            cg = orc.clip_per_tensor(cg, self.cfg["mixer_clip"])
            ag = orc.clip_per_tensor(ag, self.cfg["actor_clip"])
        self.copt.step(cg)
        self.aopt.step(ag)
        return mixer.item(), actor.item()

    def weights(self):
        w = OrderedDict((k, v.detach().numpy().astype(np.float64)) for k, v in self.wa.items())
        w.update((k, v.detach().numpy().astype(np.float64)) for k, v in self.wc.items())
        return w

    def slots(self):
        """{name: slot}: the agent's RMSProp ms, the critic's Adam (m, v)."""
        out = OrderedDict((k, ms.detach().numpy()) for k, ms in zip(self.wa, self.aopt.ms))
        out.update((k, (m.detach().numpy(), v.detach().numpy())) for k, m, v in zip(self.wc, self.copt.m, self.copt.v))
        return out


def synth_batch(seed, B, L, n, A, o, max_ep_t, early_term=True):
    """qmix_oracle.synth_batch with the raw observations: the agent inputs are [raw obs | last action one-hot | agent id]
    as QMixAlg builds them, and raw_obs the batch's obs."""
    b = qo.synth_batch(seed, B, L, n, A, o, 1, max_ep_t, early_term)
    raw = b["obs"]
    T = L + 1
    act = np.zeros((B, T, n), np.int64)
    act[:, :-1] = b["actions"]
    last = np.zeros((B, T, n, A), np.float32)
    last[:, 1:] = np.eye(A, dtype=np.float32)[act[:, :-1]]
    ids = np.broadcast_to(np.eye(n, dtype=np.float32), (B, T, n, n))
    return dict(b, raw_obs=raw, obs=np.concatenate([raw, last, ids], -1))


def model_args(batch):
    """The batch as SCCModel.train's positional arguments."""
    return (batch["obs"], batch["raw_obs"], batch["seq_len"], batch["avail"], batch["actions"], batch["state"], batch["next_state"],
            batch["reward"], batch["terminated"], batch["mask"])
