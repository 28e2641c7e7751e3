"""Float64 restatement of MuzeroModel's training step and inference (xt/model/muzero/muzero_model.py:74-239,
muzero_utils.py), with torch autograd (test-only).

Weights are the Keras list of MuzeroBase (representation, dynamics, prediction; kernel then bias per layer) and the
networks are the engine's layer tables (xingtian_b200/model/archs.py: muzero_cnn / muzero_mlp), whose softmax heads are
linear: the softmax is applied here."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import xt_oracle as orc

WEIGHT_DECAY = 1e-4


def h(x):
    return np.sign(x) * (np.sqrt(np.abs(x) + 1) - 1) + 0.001 * x


def h_inv(x):
    return np.sign(x) * (((np.sqrt(1 + 4 * 0.001 * (np.abs(x) + 1 + 0.001)) - 1) / (2 * 0.001)) ** 2 - 1)


def support_size(vmin, vmax):
    return int(np.ceil(h(vmax - vmin))) + 1


def two_hot(x, S, vmin, vmax):
    """conver_value: [..] scalars -> [.., S] two-hot rows of h(clip(x) - min); a weight past the support is dropped."""
    x = np.asarray(x, np.float64)
    v = h(np.clip(x, vmin, vmax) - vmin)
    fl = np.floor(v)
    idx, rest = fl.astype(int), v - fl
    out = np.zeros(x.shape + (S,))
    it = np.nditer(idx, flags=["multi_index"])
    for i in it:
        k = it.multi_index
        out[k + (int(i),)] = 1 - rest[k]
        if int(i) + 1 < S:
            out[k + (int(i) + 1,)] = rest[k]
    return out


def support_value(probs, vmin, vmax):
    """value_transform for every row of probs [.., S]."""
    p = np.asarray(probs, np.float64)
    e = p @ np.arange(p.shape[-1], dtype=np.float64)
    return np.clip(h_inv(e) + vmin, vmin, vmax)


def weight_shapes(arch):
    """the Keras list's shapes of one network, kernel then bias per layer"""
    return list(orc.param_shapes(arch).values())


def param_count(arch):
    return sum(int(np.prod(s)) for s in weight_shapes(arch))


def split(archs, weights):
    """the Keras list -> per-network lists of (kernel, bias)"""
    out, i = [], 0
    for a in archs:
        n = len(a["layers"])
        out.append([(weights[i + 2 * j], weights[i + 2 * j + 1]) for j in range(n)])
        i += 2 * n
    return out


def decode_obs(x, input_dtype):
    """raw observation -> float64: an int8 observation's bytes are two's-complement values"""
    x = np.asarray(x)
    if input_dtype == "int8":
        x = np.ascontiguousarray(x).astype(np.uint8).view(np.int8)
    return x.astype(np.float64)


def forward(arch, ws, x):
    """tensors of one network (float64 torch); x is the raw observation"""
    if arch["input_dtype"] == "int8":
        x = torch.from_numpy(decode_obs(x.numpy(), "int8"))
    t = {"obs": x.to(torch.float64) * arch["scale"]}
    for (name, kind, src, sp), (W, b) in zip(arch["layers"], ws):
        inp = t[src]
        if kind == "conv":
            y = F.conv2d(inp.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1), b, stride=sp["s"]).permute(0, 2, 3, 1)
        else:
            y = inp.reshape(inp.shape[0], -1) @ W + b
        if sp.get("act") == "relu":
            y = torch.relu(y)
        t[name] = y
    return t


def scale_gradient(t, s):
    return t * s + t.detach() * (1 - s)


def cross_entropy(logits, target):
    p = torch.softmax(logits, -1)
    return torch.mean(torch.mean(-target * torch.log(p + 1e-10), -1))


def train_loss(archs, params, obs, action, tv, tr, tp, K, vrange, rrange):
    """the loss of build_train_graph (muzero_model.py:103-140) without the weight-decay constant"""
    rep_a, dyn_a, pred_a = archs
    rep_w, dyn_w, pred_w = split(archs, params)
    A = tp.shape[-1]
    Sv, Sr = pred_a["layers"][-1][3]["n"], dyn_a["layers"][-1][3]["n"]
    tv2 = torch.from_numpy(two_hot(tv, Sv, *vrange))
    tr2 = torch.from_numpy(two_hot(tr, Sr, *rrange))
    tp = torch.as_tensor(tp, dtype=torch.float64)
    act = torch.as_tensor(np.asarray(action), dtype=torch.long)
    hid = forward(rep_a, rep_w, torch.as_tensor(obs))[rep_a["outputs"][0]]
    po = forward(pred_a, pred_w, hid)
    loss = cross_entropy(po["out_p"], tp[:, 0]) + cross_entropy(po["out_v"], tv2[:, 0])
    for i in range(K):
        x = torch.cat([hid, F.one_hot(act[:, i], A).to(torch.float64)], -1)
        do = forward(dyn_a, dyn_w, x)
        hid = do["out_h"]
        po = forward(pred_a, pred_w, hid)
        hid = scale_gradient(hid, 0.5)
        l = cross_entropy(do["out_r"], tr2[:, i]) + cross_entropy(po["out_p"], tp[:, i + 1]) + cross_entropy(po["out_v"], tv2[:, i + 1])
        loss = loss + scale_gradient(l, 1.0 / K)
    return loss


class Learner(object):
    """MuzeroModel.train in float64: the loss above, tf.train.AdamOptimizer(lr), the decay constant of the initial weights"""

    def __init__(self, archs, weights, K, vrange, rrange, lr=1e-3):
        self.archs, self.K, self.vrange, self.rrange, self.lr = archs, K, vrange, rrange, lr
        self.params = [torch.tensor(np.asarray(w, np.float64), requires_grad=True) for w in weights]
        self.decay = WEIGHT_DECAY * sum(0.5 * float(np.sum(np.square(np.asarray(w, np.float64)))) for w in weights)
        self.m = [torch.zeros_like(p) for p in self.params]
        self.v = [torch.zeros_like(p) for p in self.params]
        self.t = 0

    def grads(self, obs, action, tv, tr, tp):
        for p in self.params:
            p.grad = None
        loss = train_loss(self.archs, self.params, obs, action, tv, tr, tp, self.K, self.vrange, self.rrange)
        loss.backward()
        return float(loss) + self.decay, [p.grad.detach().clone() for p in self.params]

    def train(self, obs, action, tv, tr, tp):
        loss, g = self.grads(obs, action, tv, tr, tp)
        self.t += 1
        b1, b2, eps = 0.9, 0.999, 1e-8
        lr_t = self.lr * np.sqrt(1 - b2 ** self.t) / (1 - b1 ** self.t)
        with torch.no_grad():
            for p, gi, m, v in zip(self.params, g, self.m, self.v):
                m.mul_(b1).add_((1 - b1) * gi)
                v.mul_(b2).add_((1 - b2) * gi * gi)
                p.sub_(lr_t * m / (torch.sqrt(v) + eps))
        return loss, g

    def weights(self):
        return [p.detach().numpy().copy() for p in self.params]


def initial_inference(archs, weights, obs, vrange):
    rep_a, dyn_a, pred_a = archs
    rep_w, _, pred_w = split(archs, [torch.as_tensor(np.asarray(w, np.float64)) for w in weights])
    with torch.no_grad():
        hid = forward(rep_a, rep_w, torch.as_tensor(obs))[rep_a["outputs"][0]]
        po = forward(pred_a, pred_w, hid)
    value = support_value(torch.softmax(po["out_v"], -1).numpy(), *vrange)
    return value, torch.softmax(po["out_p"], -1).numpy(), hid.numpy()


def recurrent_inference(archs, weights, hidden, action, vrange, rrange):
    rep_a, dyn_a, pred_a = archs
    _, dyn_w, pred_w = split(archs, [torch.as_tensor(np.asarray(w, np.float64)) for w in weights])
    A = pred_a["layers"][1][3]["n"]
    with torch.no_grad():
        x = torch.cat([torch.as_tensor(np.asarray(hidden, np.float64)),
                       F.one_hot(torch.as_tensor(np.asarray(action), dtype=torch.long), A).to(torch.float64)], -1)
        do = forward(dyn_a, dyn_w, x)
        po = forward(pred_a, pred_w, do["out_h"])
    value = support_value(torch.softmax(po["out_v"], -1).numpy(), *vrange)
    reward = support_value(torch.softmax(do["out_r"], -1).numpy(), *rrange)
    return value, reward, torch.softmax(po["out_p"], -1).numpy(), do["out_h"].numpy()
