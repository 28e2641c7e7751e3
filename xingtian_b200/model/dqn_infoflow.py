"""DqnInfoFlowModel on the CUDA engine (xt/model/dqn/dqn_rec_model.py): the InfoFlow recommender's Q network.

A user, the ids of 5 clicked and 5 viewed items (each item item_dim ids) and one candidate item go through a frozen
Embedding; the two histories through one Keras GRU each; [user | h_click | h_noclick | item] through dense(128, relu),
dense_1(128, relu) and q_value(1, last_activate).  The weights are one flat buffer [gru | gru_1 | dense | dense_1 |
q_value] that the optimiser (Keras Adam, lr 0.001) steps; the embedding table is a buffer of its own.  The training step
(xtb_infoflow_train) and predict (xtb_infoflow_predict) run in libxtb200.

Stated assumptions, as TensorFlow is not available to pin them:
  - Embedding's mask_zero has no numeric effect: Flatten and Reshape drop the mask before anything could consume it
    (the GRUs see no mask), so id 0 looks up row 0 like any other id.
  - get_weights() lists the variables as TF 1.15's Network.weights does, trainable first: gru (kernel,
    recurrent_kernel, bias), gru_1, dense, dense_1, q_value (kernel, bias each), then the frozen Emb/embeddings.
    set_weights checks every shape, so a different order fails loudly instead of assigning wrong arrays."""
import ctypes as C
import math
import os
from collections import OrderedDict

import numpy as np
import torch

from .. import capi
from ..capi import check
from ..engine import Adam, Net, _ptr, stage_h2d, stream_ptr
from ..registry import Registers
from .base import XTModel, check_keep_model
from .impala_keras import fit_order

N_HISTORY = 5          # n_history_click = n_history_no_click = 5
HIDDEN = 128           # Dense(128, relu) twice
_ALIGN = 64            # every slice of the weight buffer starts 256-byte aligned
MAX_GRU_UNITS = 137    # item_dim * emb_dim: the GRU kernels keep both recurrent blocks in shared memory
STATE_KEYS = ("user_input", "history_click", "history_no_click", "item_input")


def _align(x):
    return (x + _ALIGN - 1) // _ALIGN * _ALIGN


def _pow2(n):
    return 1 << max(0, int(n) - 1).bit_length()


def orthogonal(rng, shape):
    """tf.orthogonal_initializer (gain 1) on a 2-D shape: QR of a standard-normal matrix with the signs of R's
    diagonal folded into Q."""
    rows, cols = shape
    a = rng.standard_normal((max(rows, cols), min(rows, cols)))
    q, r = np.linalg.qr(a)
    q = q * np.sign(np.diag(r))
    if rows < cols:
        q = q.T
    return q.reshape(shape).astype(np.float32)


def ids_int32(x, vocab, name):
    """Keras Embedding's cast of the ids to int32 (floats truncate toward zero), checked against [0, vocab)."""
    a = np.asarray(x)
    a = a.astype(np.int32) if a.dtype != np.int32 else a
    if a.size and (a.min() < 0 or a.max() >= vocab):
        raise ValueError("{}: ids must be in [0, {}) after the int32 cast".format(name, vocab))
    return a


@Registers.model
class DqnInfoFlowModel(XTModel):
    """DqnInfoFlowModel (dqn_rec_model.py:29-201)."""

    def __init__(self, model_info):
        self.state_dim = model_info["state_dim"]
        self.action_dim = model_info["action_dim"]
        self.learning_rate = 0.001
        self.vocab_size = int(model_info["vocab_size"])
        self.emb_dim = int(model_info["emb_dim"])
        self.user_dim = int(model_info["user_dim"])
        self.item_dim = int(model_info["item_dim"])
        self.input_type = model_info["input_type"]
        self.embeddings = model_info["embeddings"]
        self.last_act = model_info["last_activate"]
        if self.last_act not in capi.ACT:
            raise KeyError("last_activate {!r} is not one of {}".format(self.last_act, sorted(k for k in capi.ACT if k)))
        self.units = self.item_dim * self.emb_dim
        if min(self.vocab_size, self.emb_dim, self.user_dim, self.item_dim) < 1:
            raise ValueError("vocab_size, emb_dim, user_dim and item_dim must be positive")
        if self.units > MAX_GRU_UNITS:
            raise ValueError("item_dim x emb_dim = {} GRU units: at most {} are supported".format(self.units, MAX_GRU_UNITS))
        table = np.loadtxt(self.embeddings, delimiter=",", dtype=float)
        self._table_host = np.asarray(table, np.float32).reshape(self.vocab_size, self.emb_dim)
        self.n_history_click = self.n_history_no_click = N_HISTORY
        super().__init__(model_info)

    # ---- construction ---------------------------------------------------------------------------------------------
    def create_model(self, model_info):
        U, E = self.units, self.emb_dim
        self.in_width = self.user_dim * E + 3 * U
        head_a = dict(input_dtype="float32", state_dim=(self.in_width,), scale=1.0, layers=[
            ("dense", "dense", "obs", dict(n=HIDDEN, act="relu")),
            ("dense_1", "dense", "dense", dict(n=HIDDEN, act="relu")),
            ("q_value", "dense", "dense_1", dict(n=1, act=self.last_act)),
        ])
        self.head = Net(head_a, max_batch=256, device=self.device)
        gru = lambda: [("kernel", (U, 3 * U)), ("recurrent_kernel", (U, 3 * U)), ("bias", (3 * U,))]
        self.vars = OrderedDict()    # TF variable name -> (offset, shape) in the weight buffer, in variable order
        off, self.gru_offs = 0, []
        for scope in ("gru", "gru_1"):
            self.gru_offs.append(off)
            for name, shape in gru():
                self.vars[scope + "/" + name] = (off, shape)
                off += int(np.prod(shape))
            off = _align(off)
        self.head_off = off
        for name, (o, shape) in self.head.ptable.items():
            self.vars[name] = (self.head_off + o, shape)
        self.n_params = self.head_off + self.head.n_params
        dev = self.device
        self.params = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.table = torch.from_numpy(self._table_host).to(dev)
        self._init_weights()
        self.head.bind_to(self.params[self.head_off:], self.grads[self.head_off:])
        self.head.params_changed()
        starts = [o for o, _ in self.vars.values()] + [self.n_params]
        flat = _Flat(self.params, self.n_params, dev, starts)
        self.opt = Adam.keras(flat, self.learning_rate)
        self._natives = {}
        self._bufs = {}
        self.net = self.head
        return self.head

    def _init_weights(self):
        """Keras initialisers from the model's init generator: glorot_uniform kernels, orthogonal recurrent kernels,
        zero biases."""
        host = np.zeros(self.n_params, np.float32)
        rng = self._init_rng
        for name, (off, shape) in self.vars.items():
            size = int(np.prod(shape))
            if name.endswith("recurrent_kernel"):
                host[off:off + size] = orthogonal(rng, shape).reshape(-1)
            elif name.endswith("kernel"):
                lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                host[off:off + size] = rng.uniform(-lim, lim, size=size).astype(np.float32)
        self.params.copy_(torch.from_numpy(host))

    def _native(self, batch):
        """The native object of training batch `batch` (predict uses any)."""
        if batch is None:
            batch = next(iter(self._natives), 1)
        h = self._natives.get(batch)
        if h is None:
            d = capi.InfoflowDesc()
            d.user_dim, d.item_dim, d.emb_dim, d.vocab = self.user_dim, self.item_dim, self.emb_dim, self.vocab_size
            d.batch, d.last_act, d.gamma = int(batch), capi.ACT[self.last_act], float(getattr(self, "_gamma", 0.0))
            d.gru_off, d.gru1_off, d.head_off = self.gru_offs[0], self.gru_offs[1], self.head_off
            d.table = self.table.data_ptr()
            h = C.c_void_p()
            with torch.cuda.device(self.device):
                check(capi.lib().xtb_infoflow_create(C.byref(d), C.byref(h)))
            self._natives[batch] = h
        return h

    def set_gamma(self, gamma):
        """The TD discount of the fused step (DQNInfoFlowAlg's gamma): the native objects are rebuilt with it."""
        self._gamma = float(gamma)
        for h in self._natives.values():
            capi.lib().xtb_infoflow_destroy(h)
        self._natives = {}

    def __del__(self):
        try:
            for h in getattr(self, "_natives", {}).values():
                capi.lib().xtb_infoflow_destroy(h)
            self._natives = {}
        except Exception:
            pass

    # ---- weights ----------------------------------------------------------------------------------------------------
    def variables(self):
        """{TF variable name: ndarray} of every variable, the frozen table included (the .npz checkpoint's keys)."""
        host = self.params.detach().cpu().numpy()
        out = OrderedDict([("Emb/embeddings", self.table.detach().cpu().numpy().copy())])
        for name, (o, s) in self.vars.items():
            out[name] = host[o:o + int(np.prod(s))].reshape(s).copy()
        return out

    def _order(self):
        return list(self.vars) + ["Emb/embeddings"]

    def _shape(self, name):
        return (self.vocab_size, self.emb_dim) if name == "Emb/embeddings" else tuple(self.vars[name][1])

    def get_weights(self):
        """model.get_weights(): the Keras list (see the module docstring for its order)."""
        v = self.variables()
        return [v[k] for k in self._order()]

    def set_weights(self, weights):
        """model.set_weights(list), or TFVariables.set_weights({variable name: array}) when `weights` is a dict (names
        it does not hold are ignored; KeyError when it holds none).  Every shape is checked (ValueError)."""
        if isinstance(weights, dict):
            items = [(k, v) for k, v in weights.items() if k in self.vars or k == "Emb/embeddings"]
            if not items:
                raise KeyError("NO node's weights could assign in self.graph {} vs {}".format(self._order(), list(weights.keys())))
        else:
            weights = list(weights)
            if len(weights) != len(self._order()):
                raise ValueError("set_weights: {} arrays for {} variables".format(len(weights), len(self._order())))
            items = list(zip(self._order(), weights))
        arrays = []
        for name, value in items:
            v = np.asarray(value, dtype=np.float32)
            if tuple(v.shape) != self._shape(name):
                raise ValueError("weight {}: shape {} != {}".format(name, v.shape, self._shape(name)))
            arrays.append((name, v))
        host = self.params.detach().cpu().numpy().copy()
        for name, v in arrays:
            if name == "Emb/embeddings":
                self.table.copy_(torch.from_numpy(np.ascontiguousarray(v)))
            else:
                off, _ = self.vars[name]
                host[off:off + v.size] = v.reshape(-1)
        self.params.copy_(torch.from_numpy(host))
        self.head.params_changed()

    def save_model(self, file_name):
        """model.py:104-119 with actor_var: every variable, the table included, as file_name + ".npz"."""
        if self.max_to_keep > -1:
            check_keep_model(os.path.dirname(file_name), self.max_to_keep)
        np.savez(file_name + ".npz", **self.variables())
        return file_name + ".npz"

    def load_model(self, model_name):
        """dqn_rec_model.py:195-201 for .npz checkpoints (the Keras .h5 form is not supported)."""
        if not str(model_name).endswith(".npz"):
            raise ValueError("load_model: only .npz checkpoints are supported, got {}".format(model_name))
        with np.load(model_name) as f:
            self.set_weights(OrderedDict((k, f[k]) for k in f.files))

    # ---- device staging ---------------------------------------------------------------------------------------------
    def _ids(self, key, n_words):
        """Grow-only int32 device buffer `key` of at least n_words (power-of-two capacity)."""
        b = self._bufs.get(key)
        if b is None or b.numel() < n_words:
            b = torch.zeros(_pow2(max(n_words, 64)), dtype=torch.int32, device=self.device)
            self._bufs[key] = b
        return b

    def _head_rows(self, rows):
        if rows > self.head.max_batch:
            self.head.ensure_batch(_pow2(rows))
            self.head.params_changed()

    def state_ids(self, state):
        """The tiled dict form {user_input, history_click, history_no_click, item_input} -> int32 arrays, checked."""
        shapes = dict(user_input=self.user_dim, history_click=N_HISTORY * self.item_dim,
                      history_no_click=N_HISTORY * self.item_dim, item_input=self.item_dim)
        out = []
        n = None
        for k in STATE_KEYS:
            a = ids_int32(state[k], self.vocab_size, k)
            a = a.reshape(a.shape[0] if a.ndim else 1, -1)
            if a.shape[1] != shapes[k] or (n is not None and a.shape[0] != n):
                raise ValueError("{}: [N, {}] ids expected, got {}".format(k, shapes[k], a.shape))
            n = a.shape[0]
            out.append(np.ascontiguousarray(a))
        return out

    # ---- predict / train --------------------------------------------------------------------------------------------
    def predict(self, state):
        """dqn_rec_model.py:156-169: Q values [N] float32 of N rows in the tiled dict form."""
        parts = self.state_ids(state)
        n = parts[0].shape[0]
        if n == 0:
            return np.zeros(0, np.float32)
        packed = np.concatenate([p.reshape(-1) for p in parts])
        buf = self._ids("predict", packed.size)
        stage_h2d(buf[:packed.size], packed, np.int32)
        q = self._bufs.get("q")
        if q is None or q.numel() < n:
            q = self._bufs["q"] = torch.empty(_pow2(n), dtype=torch.float32, device=self.device)
        self._head_rows(n)
        offs = np.cumsum([0] + [p.size for p in parts])
        base = buf.data_ptr()
        ptrs = [C.c_void_p(base + 4 * int(o)) for o in offs[:4]]
        check(capi.lib().xtb_infoflow_predict(self._native(None), self.head.handle, *ptrs, int(n), _ptr(q),
                                              1 if self.use_graph else 0, stream_ptr()))
        return q[:n].cpu().numpy()

    def train(self, state, label, batch_size, verbose=False):
        """dqn_rec_model.py:147-154: model.fit(state, label, batch_size) with N <= batch_size rows is one step of Keras
        Adam on mse; its shuffle advances np.random once (it only reorders the step's sum).  Returns the loss before
        the update."""
        user, click, noclick, item = self.state_ids(state)
        n = user.shape[0]
        y = np.asarray(label, np.float32).reshape(-1)
        if n < 1 or n > int(batch_size) or y.size != n:
            raise ValueError("train: 1 <= N <= batch_size rows and N labels expected (N = {}, batch_size {}, {} labels)".format(
                n, batch_size, y.size))
        fit_order(n)
        lab = self._bufs.get(("label", n))
        if lab is None:
            lab = self._bufs[("label", n)] = torch.empty(n, dtype=torch.float32, device=self.device)
        stage_h2d(lab, y, np.float32)
        return self._train_packed(dict(user=user, click=click, noclick=noclick, item=item), label=lab)

    def train_transitions(self, batch, gamma):
        """One DQNInfoFlowAlg step on the packed minibatch `batch` (see DQNInfoFlowAlg.pack): the targets from the
        online net's Q over every candidate, then the fit step -> loss.  The caller advances np.random for fit's
        shuffle."""
        if getattr(self, "_gamma", None) != float(gamma):
            self.set_gamma(gamma)
        return self._train_packed(batch)

    def _train_packed(self, b, label=None, target_out=None):
        B = b["user"].shape[0]
        full = label is None
        n_cand = int(b["cand_off"][-1]) if full else 0
        cap = _pow2(max(n_cand, B))
        cap = max(cap, self._bufs.get(("cap", B), 0))
        self._bufs[("cap", B)] = cap
        # one int32 upload: [reward (float64 pairs) | user | click | noclick | item | next_* | cand_off | done | cand_item]
        order = ["user", "click", "noclick", "item"]
        if full:
            order += ["next_user", "next_click", "next_noclick", "cand_off", "done"]
        parts = [np.asarray(b["reward"], np.float64).view(np.int32)] if full else []
        parts += [np.asarray(b[k], np.int32).reshape(-1) for k in order]
        if full:
            ci = np.zeros(cap * self.item_dim, np.int32)
            ci[:n_cand * self.item_dim] = np.asarray(b["cand_item"], np.int32).reshape(-1)
            parts.append(ci)
        packed = np.concatenate(parts)
        buf = self._ids(("train", full), packed.size)
        stage_h2d(buf[:packed.size], packed, np.int32)
        base, pos = buf.data_ptr(), 0
        bt = capi.InfoflowBatch()
        if full:
            bt.reward = base
            pos = 2 * B
        for k, p in zip(order + (["cand_item"] if full else []), parts[1 if full else 0:]):
            setattr(bt, k, base + 4 * pos)
            pos += p.size
        if not full:
            bt.label = label.data_ptr()
        bt.n_cand, bt.cand_cap = n_cand, cap
        self._head_rows(cap)
        loss = self._bufs.get("loss")
        if loss is None:
            loss = self._bufs["loss"] = torch.zeros(1, dtype=torch.float32, device=self.device)
        check(capi.lib().xtb_infoflow_train(self._native(B), self.head.handle, self.opt.handle, C.byref(bt), _ptr(loss),
                                            _ptr(target_out), 1 if self.use_graph else 0, stream_ptr()))
        return float(loss.cpu()[0])


class _Flat(object):
    """The optimiser's view of the weight buffer: one segment per variable."""

    def __init__(self, params, n_params, device, starts):
        self.params, self.n_params, self.device, self._starts = params, n_params, device, starts

    def segment_offsets(self):
        return self._starts
