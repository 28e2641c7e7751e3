"""Thin Python owner of one libxtb200 network: allocates storage as torch tensors (device memory
and streams are PyTorch plumbing), binds it through the C-ABI and exposes named views."""
import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import capi
from .capi import check


def _ptr(t):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def stage_h2d(dst, arr, np_dtype):
    """Copy one host (pageable) array into the contiguous device tensor `dst` through the library's staged copy
    (`xtb_copy_h2d_staged`: worker threads fill a pinned ring while earlier chunks are in flight); asynchronous on the
    current stream, the source may be reused as soon as the call returns."""
    import numpy as np
    a = np.ascontiguousarray(arr, dtype=np_dtype).reshape(tuple(dst.shape))
    if not dst.is_contiguous():
        raise ValueError("staging target must be contiguous")
    capi.check(capi.lib().xtb_copy_h2d_staged(_ptr(dst), a.ctypes.data, a.nbytes, stream_ptr()))


class DeviceStore(object):
    """Grow-only named device arrays: field `name` is [capacity, *row_shape] of its dtype, an attribute of the store.
    The arrays keep their addresses until the next growth, so the CUDA graphs captured on them are replayed instead of
    re-captured.  `n` is the number of valid rows, the ones a growth keeps."""

    def __init__(self, device, **fields):
        self.device, self.fields = device, fields    # name -> (row shape, torch dtype)
        self.capacity = self.n = 0
        for name in fields:
            setattr(self, name, None)

    def reserve(self, rows):
        """Make room for `rows` rows: a growth reallocates every array to max(rows, 2 x capacity) rows and copies the
        first `n` rows over."""
        if self.n > self.capacity:
            raise ValueError("store holds %d rows but %d are marked valid" % (self.capacity, self.n))
        if rows <= self.capacity:
            return
        cap = max(int(rows), 2 * self.capacity)
        for name, (shape, dtype) in self.fields.items():
            new = torch.empty((cap,) + tuple(shape), dtype=dtype, device=self.device)
            if self.n:
                new[:self.n].copy_(getattr(self, name)[:self.n])
            setattr(self, name, new)
        self.capacity = cap


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("xingtian_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")


def net_desc(arch):
    """The xtb_net_desc of `arch` (layers = list of (name, kind, src_name, spec), see Net); xtb_net_create plans it on
    the host."""
    tid = {n: i for i, n in enumerate(["obs"] + [l[0] for l in arch["layers"]])}
    desc = capi.NetDesc()
    desc.input_u8 = {"uint8": 1, "int8": 2}.get(arch["input_dtype"], 0)
    desc.scale = float(arch["scale"])
    sd = tuple(arch["state_dim"])
    desc.in_h, desc.in_w, desc.in_c = (sd if len(sd) == 3 else (1, 1, int(np.prod(sd))))
    desc.n_layers = len(arch["layers"])
    if desc.n_layers > capi.XTB_MAX_LAYERS:
        raise ValueError("too many layers")
    for i, (name, kind, src, sp) in enumerate(arch["layers"]):
        ld = desc.layers[i]
        if kind == "dueling":
            ld.kind, ld.src, ld.k, ld.act = capi.DUELING, tid[src[0]], tid[src[1]], capi.ACT[None]
            continue
        if kind == "logstd":
            ld.kind, ld.src, ld.cout, ld.act = capi.LOGSTD, 0, sp["n"], capi.ACT[None]
            continue
        ld.kind = capi.CONV if kind == "conv" else capi.DENSE
        ld.src = tid[src]
        ld.act = capi.ACT[sp.get("act")]
        if kind == "conv":
            ld.k, ld.stride, ld.cout = sp["k"], sp["s"], sp["cout"]
            ld.pad_same = 1 if sp["pad"] == "same" else 0
        else:
            ld.cout = sp["n"]
    return desc


class Net(object):
    """One network (layers = list of (name, kind, src_name, spec)) living in device memory.

    kind "dueling": (name, "dueling", (value_src, adv_src), {}) combines an A-wide and a 1-wide earlier tensor into
    Q = adv + (value - mean(value)); it has no parameters.
    kind "logstd": (name, "logstd", None, dict(n=A)) is a parameter-only layer (PPO's pi_logstd): A floats under the
    weight name `name` with shape (1, A); it reads and produces no tensor."""

    def __init__(self, arch, max_batch, device="cuda:0"):
        require_cuda()
        self.lib = capi.lib()
        self.arch = arch
        self.device = torch.device(device)
        self.max_batch = int(max_batch)
        self.names = ["obs"] + [l[0] for l in arch["layers"]]
        self.tid = {n: i for i, n in enumerate(self.names)}
        self._desc = net_desc(arch)
        self.handle = C.c_void_p()
        self.params = self.grads = None
        self._create(self.max_batch)
        # parameter table: tf-style name -> (offset, shape)
        self.ptable = OrderedDict()
        in_shapes = self._shapes()
        for i, (name, kind, src, sp) in enumerate(arch["layers"]):
            if kind == "dueling":
                continue
            ko, bo, kr, nc = C.c_longlong(), C.c_longlong(), C.c_int(), C.c_int()
            check(self.lib.xtb_net_layer_params(self.handle, i, C.byref(ko), C.byref(bo), C.byref(kr), C.byref(nc)))
            if kind == "logstd":
                self.ptable[name] = (ko.value, (kr.value, nc.value))
                continue
            if kind == "conv":
                kshape = (sp["k"], sp["k"], in_shapes[src][-1], sp["cout"])
            else:
                kshape = (kr.value, nc.value)
            assert int(np.prod(kshape)) == kr.value * nc.value
            self.ptable[name + "/kernel"] = (ko.value, kshape)
            self.ptable[name + "/bias"] = (bo.value, (nc.value,))

    def _create(self, max_batch):
        """(Re)create the native handle + activation workspace for `max_batch` samples; the flat
        parameter / gradient tensors are kept (their pointers never change)."""
        if self.handle.value:
            self.lib.xtb_net_destroy(self.handle)
            self.handle = C.c_void_p()
        self.max_batch = int(max_batch)
        with torch.cuda.device(self.device):
            check(self.lib.xtb_net_create(C.byref(self._desc), self.max_batch, C.byref(self.handle)))
        self.n_params = int(self.lib.xtb_net_param_count(self.handle))
        if self.params is None:
            self.params = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
            self.grads = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
        ws_bytes = int(self.lib.xtb_net_workspace_bytes(self.handle))
        self.ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device=self.device)
        self._ws_base = (self.ws.data_ptr() + 255) // 256 * 256
        with torch.cuda.device(self.device):
            check(self.lib.xtb_net_bind_stream(self.handle, _ptr(self.params), _ptr(self.grads),
                                               C.c_void_p(self._ws_base), ws_bytes, stream_ptr()))

    def bind_to(self, params, grads):
        """Rebind the network to `params` / `grads` (float32 device views of n_params floats, e.g. slices of a buffer shared
        with other networks); the workspace is kept and its contents are reset."""
        for t in (params, grads):
            if t.numel() != self.n_params or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError("bind_to needs contiguous float32 views of %d floats" % self.n_params)
        self.params, self.grads = params, grads
        ws_bytes = int(self.lib.xtb_net_workspace_bytes(self.handle))
        with torch.cuda.device(self.device):
            check(self.lib.xtb_net_bind_stream(self.handle, _ptr(self.params), _ptr(self.grads),
                                               C.c_void_p(self._ws_base), ws_bytes, stream_ptr()))

    def backward_input(self, obs, batch, heads, dobs, idx=None):
        """backward() that also writes d loss / d observation into `dobs` [batch, obs width] (xtb_net_backward_input)."""
        arr = (C.c_int32 * len(heads))(*[self.tid[h] for h in heads])
        check(self.lib.xtb_net_backward_input(self.handle, _ptr(obs), _ptr(idx), int(batch), arr, len(heads), _ptr(dobs),
                                              stream_ptr()))

    def params_changed(self):
        """Must follow every host-side write into `self.params`: refreshes the bf16 hi/lo planes the
        tensor-core kernels read (xtb_net_sync_weights)."""
        check(self.lib.xtb_net_sync_weights(self.handle, stream_ptr()))

    def load_flat(self, flat):
        """Copy a flat parameter vector (e.g. another network's `params`) into this network."""
        self.params.copy_(flat)
        self.params_changed()

    def ensure_batch(self, batch):
        if batch > self.max_batch:
            torch.cuda.current_stream().synchronize()
            self._create(batch)

    def layer_plan(self, i):
        """How the library planned layer i (xtb_net_layer_plan): kind ("conv" / "dense" / "dueling", after a VALID conv that
        covers the whole map became dense), tc, s2d, w_res, n_fwd, n_dg, R, fwd_stages, dg_stages, dg_empty_units,
        k_slices."""
        p = capi.LayerPlan()
        check(self.lib.xtb_net_layer_plan(self.handle, int(i), C.byref(p)))
        out = {name: int(getattr(p, name)) for name, _ in capi.LayerPlan._fields_}
        out["kind"] = {capi.CONV: "conv", capi.DENSE: "dense", capi.DUELING: "dueling", capi.LOGSTD: "logstd"}[p.kind]
        for k in ("tc", "s2d", "w_res"):
            out[k] = bool(out[k])
        return out

    def _shapes(self):
        shapes = {"obs": tuple(self.arch["state_dim"])}
        for name, kind, src, sp in self.arch["layers"]:
            if kind == "dueling":
                shapes[name] = shapes[src[0]]
                continue
            if kind == "logstd":
                continue
            ish = shapes[src]
            if kind == "conv":
                h, w, _ = ish
                if sp["pad"] == "same":
                    oh, ow = -(-h // sp["s"]), -(-w // sp["s"])
                else:
                    oh, ow = (h - sp["k"]) // sp["s"] + 1, (w - sp["k"]) // sp["s"] + 1
                shapes[name] = (oh, ow, sp["cout"])
            else:
                shapes[name] = (sp["n"],)
        return shapes

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                self.lib.xtb_net_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:  # interpreter shutdown
            pass

    # ---- weights (xt/model/tf_utils.py:99-128 dict format) -------------------------------
    def segment_offsets(self):
        offs = [off for off, _ in self.ptable.values()] + [self.n_params]
        return offs

    def view(self, name, flat=None):
        off, shape = self.ptable[name]
        flat = self.params if flat is None else flat
        return flat[off:off + int(np.prod(shape))].view(*shape)

    def get_weights(self, flat=None):
        host = (self.params if flat is None else flat).detach().cpu().numpy()
        out = OrderedDict()
        for name, (off, shape) in self.ptable.items():
            out[name] = host[off:off + int(np.prod(shape))].reshape(shape).copy()
        return out

    def set_weights(self, weights, flat=None):
        flat = self.params if flat is None else flat
        hit = 0
        host = flat.detach().cpu().numpy().copy()
        for name, value in weights.items():
            if name in self.ptable:
                off, shape = self.ptable[name]
                v = np.asarray(value, dtype=np.float32)
                if tuple(v.shape) != tuple(shape):
                    raise ValueError("weight %s: shape %s != %s" % (name, v.shape, shape))
                host[off:off + v.size] = v.reshape(-1)
                hit += 1
        if not hit:
            raise KeyError("NO node's weights could assign in self.graph {} vs {}".format(
                list(self.ptable.keys()), list(weights.keys())))
        flat.copy_(torch.from_numpy(host))
        if flat is self.params:
            self.params_changed()

    # ---- tensors ---------------------------------------------------------------------------
    def _wrap(self, ptr, t):
        size = int(self.lib.xtb_net_tensor_size(self.handle, t))
        off = ptr - self.ws.data_ptr()
        return self.ws[off:off + self.max_batch * size * 4].view(torch.float32).view(self.max_batch, size)

    def tensor(self, name):
        t = self.tid[name]
        return self._wrap(self.lib.xtb_net_tensor(self.handle, t), t)

    def tensor_grad(self, name):
        t = self.tid[name]
        return self._wrap(self.lib.xtb_net_tensor_grad(self.handle, t), t)

    # ---- compute ---------------------------------------------------------------------------
    def forward(self, obs, batch, idx=None, params=None):
        check(self.lib.xtb_net_forward(self.handle, _ptr(params), _ptr(obs), _ptr(idx), int(batch), stream_ptr()))

    def backward(self, obs, batch, heads, idx=None):
        arr = (C.c_int32 * len(heads))(*[self.tid[h] for h in heads])
        check(self.lib.xtb_net_backward(self.handle, _ptr(obs), _ptr(idx), int(batch), arr, len(heads), stream_ptr()))


class Adam(object):
    """tf.train.AdamOptimizer(+clip_by_global_norm) / keras Adam(clipnorm) on one flat bucket."""

    def __init__(self, net, lr, eps=1e-8, clip_mode=capi.CLIP_GLOBAL_NORM, clip=5.0, beta1=0.9, beta2=0.999):
        self.lib = capi.lib()
        self.net = net
        self.m = torch.zeros_like(net.params)
        self.v = torch.zeros_like(net.params)
        offs = net.segment_offsets()
        # kernel and bias of a layer are separate tensors for per-tensor clipping
        seg = (C.c_longlong * len(offs))(*offs)
        self.handle = C.c_void_p()
        with torch.cuda.device(net.device):
            check(self.lib.xtb_adam_create(net.n_params, lr, beta1, beta2, eps, clip_mode, clip, seg,
                                           len(offs) - 1, _ptr(self.m), _ptr(self.v), C.byref(self.handle)))

    @classmethod
    def keras(cls, net, lr, clipnorm=None):
        """keras.optimizers.Adam(lr, clipnorm): epsilon = K.epsilon() = 1e-7, each gradient tensor clipped to norm
        `clipnorm` on its own (no clipping without one)."""
        mode = capi.CLIP_PER_TENSOR if clipnorm else capi.CLIP_NONE
        return cls(net, lr, eps=1e-7, clip_mode=mode, clip=float(clipnorm or 0.0))

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                self.lib.xtb_adam_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:
            pass

    def use_rmsprop(self, decay=0.99, epsilon=0.1, centered=True):
        """tf.train.RMSPropOptimizer(lr, decay, epsilon, centered): mean-square slot starts at ones, mean-gradient (centred
        only; else None) at zeros."""
        if not centered:
            self.mean_grad = None
            check(self.lib.xtb_opt_use_rmsprop_plain(self.handle, float(decay), float(epsilon)))
            return
        self.mean_grad = torch.zeros_like(self.net.params)
        check(self.lib.xtb_opt_use_rmsprop(self.handle, _ptr(self.mean_grad), float(decay), float(epsilon)))

    def set_lr(self, lr):
        check(self.lib.xtb_adam_set_lr(self.handle, float(lr)))

    def set_decay(self, decay):
        """Keras OptimizerV2 `decay`: later steps use lr / (1 + decay * steps taken before them)."""
        check(self.lib.xtb_adam_set_decay(self.handle, float(decay)))

    def step(self, grad_scale=1.0):
        check(self.lib.xtb_adam_step_net(self.handle, self.net.handle, float(grad_scale), stream_ptr()))

    def grad_norm(self):
        p = self.lib.xtb_adam_grad_norm(self.handle)
        out = torch.empty(1, dtype=torch.float32)
        torch.cuda.current_stream().synchronize()
        check(self.lib.xtb_copy_d2h(C.c_void_p(out.data_ptr()), C.c_void_p(p), 4, stream_ptr()))
        torch.cuda.current_stream().synchronize()
        return float(out[0])


def _nccl_path():
    """libnccl of the running PyTorch (nvidia-nccl wheel); None lets the library try the loader path."""
    import os
    try:
        import nvidia.nccl as pkg
        for base in list(getattr(pkg, "__path__", [])):
            cand = os.path.join(base, "lib", "libnccl.so.2")
            if os.path.exists(cand):
                return cand
    except Exception:
        pass
    return None


class GradComm(object):
    """Data-parallel learner (SURVEY 8(e)) with the library's own NCCL communicator: the gradient all-reduce is issued
    by the fused training loops themselves, inside their CUDA graph, the big dense bucket under the conv backward.
    torch.distributed is only the out-of-band channel that ships the NCCL unique id from rank 0."""

    def __init__(self, group=None, device=None):
        import torch.distributed as dist
        self.lib = capi.lib()
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        path = _nccl_path()
        cpath = path.encode() if path else None
        buf = (C.c_ubyte * 128)()
        if self.rank == 0:
            check(self.lib.xtb_comm_unique_id(cpath, buf))
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        backend = dist.get_backend(group)
        t = torch.tensor(list(bytes(buf)), dtype=torch.uint8, device=dev if backend == "nccl" else "cpu")
        dist.broadcast(t, src=0, group=group)
        ident = (C.c_ubyte * 128)(*t.cpu().tolist())
        self.handle = C.c_void_p()
        with torch.cuda.device(dev):
            check(self.lib.xtb_comm_create(cpath, ident, self.rank, self.world, C.byref(self.handle)))
        check(self.lib.xtb_set_grad_comm(self.handle))

    def all_reduce_(self, tensor):
        """In-place sum of a float32 device tensor over the ranks (utility; the training loops do their own)."""
        check(self.lib.xtb_comm_allreduce(self.handle, _ptr(tensor), tensor.numel(), stream_ptr()))
        return tensor

    def detach(self):
        """Stop all-reducing (single-rank work on this process), keep the communicator alive."""
        check(self.lib.xtb_set_grad_comm(None))

    def attach(self):
        check(self.lib.xtb_set_grad_comm(self.handle))

    def close(self):
        """Collective: every rank must call it (the graphs that captured this communicator are destroyed first)."""
        if self.handle.value:
            check(self.lib.xtb_set_grad_comm(None))
            self.lib.xtb_comm_destroy(self.handle)
            self.handle = C.c_void_p()
