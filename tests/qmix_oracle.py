"""Float64 restatement of QMixModel's train graph (xt/model/qmix/qmix_tf.py) and its explore step, with autograd
gradients, per-variable clip_by_norm and centred RMSProp (oracle.xt_oracle.clip_per_tensor / TFRMSProp).  The arithmetic
type follows oracle.xt_oracle.precision: "f64" is the yardstick, "f32" the size of fp32 rounding."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import xt_oracle as orc

GATES_K, GATES_B = "rnn/gru_cell/gates/kernel", "rnn/gru_cell/gates/bias"
CAND_K, CAND_B = "rnn/gru_cell/candidate/kernel", "rnn/gru_cell/candidate/bias"
MIX_LAYERS = ("hyper_w1/dense", "hyper_w1/dense_1", "hyper_b1/dense", "hyper_w_final/dense", "hyper_w_final/dense_1",
              "val_for_bias/dense", "val_for_bias/dense_1")


def _t(x):
    return torch.as_tensor(np.asarray(x), dtype=orc._PREC["t"])


def gru_cell(x, h, w):
    """tf.nn.rnn_cell.GRUCell (TF 1.15): [r|u] = sigmoid([x, h] Wg + bg), c = tanh([x, r h] Wc + bc), h' = u h + (1-u) c."""
    H = h.shape[-1]
    ru = torch.sigmoid(torch.cat([x, h], -1) @ w[GATES_K] + w[GATES_B])
    r, u = ru[..., :H], ru[..., H:]
    c = torch.tanh(torch.cat([x, r * h], -1) @ w[CAND_K] + w[CAND_B])
    return u * h + (1 - u) * c


def dynamic_rnn(x, lens, w, h0=None):
    """tf.nn.dynamic_rnn over x [S, T, H]: outputs past a sequence's length are zero and its state stays put."""
    S, T, H = x.shape
    h = torch.zeros(S, H, dtype=x.dtype) if h0 is None else h0
    outs = []
    lens = torch.as_tensor(np.asarray(lens))
    for t in range(T):
        hn = gru_cell(x[:, t], h, w)
        live = (t < lens).unsqueeze(-1)
        h = torch.where(live, hn, h)
        outs.append(torch.where(live, hn, torch.zeros_like(hn)))
    return torch.stack(outs, 1), h


def agent_forward(w, obs, lens, h0=None):
    """build_agent_net on obs [B, T, n, obs] -> (Q [B, T, n, A], final state [B n, H])."""
    B, T, n, _ = obs.shape
    fc1 = torch.relu(obs @ w["dense/kernel"] + w["dense/bias"])
    H = fc1.shape[-1]
    seq = fc1.permute(0, 2, 1, 3).reshape(B * n, T, H)
    out, hT = dynamic_rnn(seq, lens, w, h0)
    out = out.reshape(B, n, T, H).permute(0, 2, 1, 3)
    return out @ w["dense_1/kernel"] + w["dense_1/bias"], hT


def _dense(w, name, x, relu=False):
    y = x @ w[name + "/kernel"] + w[name + "/bias"]
    return torch.relu(y) if relu else y


def mixer(w, q, states):
    """_build_mix_net2: q [B, L, n], states [B, L, sd] -> q_tot [B, L]."""
    B, L, n = q.shape
    s = states.reshape(B * L, -1)
    w1 = torch.abs(_dense(w, "hyper_w1/dense_1", _dense(w, "hyper_w1/dense", s, True))).reshape(-1, n, w["hyper_b1/dense/bias"].shape[0])
    b1 = _dense(w, "hyper_b1/dense", s).unsqueeze(1)
    hidden = torch.nn.functional.elu(q.reshape(-1, 1, n) @ w1 + b1)
    wf = torch.abs(_dense(w, "hyper_w_final/dense_1", _dense(w, "hyper_w_final/dense", s, True))).unsqueeze(-1)
    v = _dense(w, "val_for_bias/dense_1", _dense(w, "val_for_bias/dense", s, True)).reshape(-1, 1, 1)
    return (hidden @ wf + v).reshape(B, L)


def first_argmax(x):
    """tf.argmax over the last axis: the lowest index among equal maxima."""
    mx = x.max(-1, keepdim=True).values
    idx = torch.arange(x.shape[-1]).expand_as(x)
    return torch.where(x == mx, idx, x.shape[-1]).min(-1).values


def count_ties(q, avail, mask):
    """Masked-in (episode, step t, agent) rows whose step t + 1 Q values (q [B, T, n, A], avail [B, T, n, A], mask
    [B, T - 1]) have two or more available actions at the maximum over the available ones: the rows where the TD
    target's argmax (double Q) or max has a tie to break."""
    q, av = np.asarray(q)[:, 1:], np.asarray(avail)[:, 1:] > 0
    q = np.where(av, q, -np.inf)
    at_max = av & (q == q.max(-1, keepdims=True))
    return int(((at_max.sum(-1) >= 2) & (np.asarray(mask)[..., None] > 0)).sum())


def td_loss(w, wt, batch, gamma, double_q):
    """The loss of build_train_graph on a host batch (dict of arrays, the QMixModel.train arguments)."""
    obs, avail = _t(batch["obs"]), _t(batch["avail"])
    lens = batch["seq_len"]
    act = torch.as_tensor(np.asarray(batch["actions"]), dtype=torch.int64)
    mac, _ = agent_forward(w, obs, lens)
    with torch.no_grad():
        tmac, _ = agent_forward(wt, obs, lens)
    chosen = torch.gather(mac[:, :-1], -1, act.unsqueeze(-1)).squeeze(-1)
    unavail = avail[:, 1:] == 0
    tmac = torch.where(unavail, torch.full_like(tmac[:, 1:], -999999.0), tmac[:, 1:])
    if double_q:
        e = torch.where(unavail, torch.full_like(tmac, -999999.0), mac[:, 1:].detach())
        tmax = torch.gather(tmac, -1, first_argmax(e).unsqueeze(-1)).squeeze(-1)
    else:
        tmax = tmac.max(-1).values
    q_tot = mixer(w, chosen, _t(batch["state"]))
    with torch.no_grad():
        tq_tot = mixer(wt, tmax, _t(batch["next_state"]))
    mask = _t(batch["mask"])
    targets = _t(batch["reward"]) + gamma * (1 - _t(batch["terminated"])) * tq_tot
    mtd = (q_tot - targets) * mask
    return (mtd ** 2).sum() / mask.sum()


class QmixLearner(object):
    """Eval / target weights {name: tensor} of the model's variable tables, RMSProp(lr, 0.95, 1.5e-7) with
    clip_by_norm(grad_norm_clip) of every gradient."""

    def __init__(self, eval_w, target_w, lr, grad_norm_clip, gamma, double_q):
        self.w = OrderedDict((k, _t(v).clone().requires_grad_(True)) for k, v in eval_w.items())
        self.wt = OrderedDict((k, _t(v)) for k, v in target_w.items())
        self.opt = orc.TFRMSProp(list(self.w.values()), lr, decay=0.95, eps=1.5e-7)
        self.clip, self.gamma, self.double_q = grad_norm_clip, gamma, double_q

    def step(self, batch):
        loss = td_loss(self.w, self.wt, batch, self.gamma, self.double_q)
        grads = torch.autograd.grad(loss, list(self.w.values()), allow_unused=True)
        grads = [torch.zeros_like(p) if g is None else g for p, g in zip(self.w.values(), grads)]
        self.opt.step(orc.clip_per_tensor(grads, self.clip))
        return loss.item()

    def assign_targets(self):
        self.wt = OrderedDict((k, v.detach().clone()) for k, v in self.w.items())

    def slots(self):
        """{name: (ms, mg)} of the RMSProp slots."""
        return OrderedDict((k, (ms.detach().numpy(), mg.detach().numpy())) for k, ms, mg in zip(self.w, self.opt.ms, self.opt.mg))


def synth_batch(seed, B, L, n, A, obs_dim, state_dim, max_ep_t, early_term=True):
    """A batch as QMixAlg.train hands it over: episodes filled up to random lengths <= max_ep_t (one of them exactly
    max_ep_t), zero padding beyond, some episodes terminated early, avail masks with unavailable actions (padding rows all
    unavailable, as the zero-filled buffer has them), mask = filled[:, :-1] with mask[:, 1:] *= 1 - terminated[:, :-1]."""
    rng = np.random.default_rng(seed)
    T = L + 1
    filled = np.zeros((B, T), np.float32)
    lens = rng.integers(1, max_ep_t + 1, size=B)
    lens[0] = max_ep_t
    obs = np.zeros((B, T, n, obs_dim), np.float32)
    state = np.zeros((B, T, state_dim), np.float32)
    avail = np.zeros((B, T, n, A), np.int32)
    actions = np.zeros((B, T, n), np.int64)
    reward = np.zeros((B, T), np.float32)
    term = np.zeros((B, T), np.uint8)
    for b in range(B):
        m = int(lens[b])
        filled[b, :m] = 1
        obs[b, :m] = rng.normal(size=(m, n, obs_dim))
        state[b, :m] = rng.normal(size=(m, state_dim))
        av = (rng.random((m, n, A)) < 0.6).astype(np.int32)
        av[..., 0] = 1
        avail[b, :m] = av
        for t in range(m):
            for a in range(n):
                actions[b, t, a] = rng.choice(np.flatnonzero(av[t, a]))
        reward[b, :m] = rng.normal(size=m)
        if early_term and m > 1 and b % 2 == 1:
            term[b, m - 2] = 1
    mask = filled[:, :-1].copy()
    terminated = term[:, :-1].astype(np.float32)
    mask[:, 1:] = mask[:, 1:] * (1 - terminated[:, :-1])
    return dict(obs=obs, seq_len=np.full(B * n, max_ep_t, np.int32), avail=avail.astype(np.float32), actions=actions[:, :-1],
                state=state[:, :-1], next_state=state[:, 1:], reward=reward[:, :-1], terminated=terminated, mask=mask)


def model_args(batch):
    """The batch as QMixModel.train's positional arguments."""
    return (batch["obs"], batch["seq_len"], batch["avail"], batch["actions"], batch["state"], batch["next_state"], batch["reward"],
            batch["terminated"], batch["mask"])
