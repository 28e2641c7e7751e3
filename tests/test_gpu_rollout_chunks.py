"""Rollout inference evaluates several steps per forward pass (as many as fit the net's max_batch rows).  Its results
must not depend on that: a T-step call gives bitwise the actions, log-probs and values of T one-step calls, leaves the
last step's pi head in rows [0, E) of its tensor, and launches one chunk's kernels per max_batch // E steps."""
import numpy as np
import pytest
import torch

from test_gpu_kernels import _keepalive, tc_mode, xb  # noqa: F401

pytestmark = pytest.mark.gpu

MAX_BATCH = 320
_MODELS = {}


def _model(kind):
    """PpoCnn Categorical (uint8 frames, A=4, relu [256]), ImpalaCnnOpt (uint8 frames, A=4) or PpoMlp DiagGaussian ([3] ->
    A=3, tanh [256, 256], separate towers), all planned for MAX_BATCH rows; one instance per kind for the module"""
    if kind not in _MODELS:
        import xingtian_b200  # noqa: F401
        from xingtian_b200.registry import Registers
        if kind == "cnn":
            info = {"state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8", "max_predict_batch": MAX_BATCH,
                    "model_config": {"BATCH_SIZE": MAX_BATCH, "hidden_sizes": [256], "action_type": "Categorical",
                                     "init_seed": 5}}
            m = Registers.model["PpoCnn"](info)
        elif kind == "impala":
            info = {"state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8", "state_mean": 0.0, "state_std": 255.0,
                    "max_batch": MAX_BATCH, "model_config": {"init_seed": 7}}
            m = Registers.model["ImpalaCnnOpt"](info)
        else:
            info = {"state_dim": [3], "action_dim": 3, "max_predict_batch": MAX_BATCH,
                    "model_config": {"BATCH_SIZE": MAX_BATCH, "hidden_sizes": [256, 256], "activation": "tanh",
                                     "VF_SHARE_LAYERS": False, "action_type": "DiagGaussian", "init_seed": 6}}
            m = Registers.model["PpoMlp"](info)
            w = m.get_weights()
            w["pi_logstd"] = np.array([[-0.3, 0.2, 0.5]], np.float32)
            m.set_weights(w)
        assert m.net.max_batch == MAX_BATCH
        _MODELS[kind] = m
    return _MODELS[kind]


def _obs(kind, E, T, seed):
    """T steps of E observations: frames env-major with a [T][E] row index (the trajectory layout), PpoMlp states
    time-major without one"""
    rng = np.random.default_rng(seed)
    if kind != "mlp":
        obs = torch.from_numpy(rng.integers(0, 256, (E * T, 84, 84, 4), dtype=np.uint8)).cuda()
        idx = (torch.arange(E, dtype=torch.int32)[None, :] * T + torch.arange(T, dtype=torch.int32)[:, None]).contiguous()
        return obs, idx.cuda()
    return torch.from_numpy(rng.standard_normal((E * T, 3)).astype(np.float32)).cuda(), None


def _outputs(m, E, T):
    shape = (T, E, m.action_dim) if m.ls_t else (T, E)
    act = torch.empty(shape, dtype=torch.float32 if m.ls_t else torch.int32, device="cuda")
    return act, torch.empty(T, E, device="cuda"), torch.empty(T, E, device="cuda")


def _pi_head(m, E):
    net = m.net
    return net.tensor(net.names[m.pi_t])[:E].cpu().numpy().copy()


def _infer(m, obs, idx, E, T, base, graph):
    """one T-step call from offset `base`: actions, log-probs, values and rows [0, E) of the pi head's tensor"""
    act, lp, val = _outputs(m, E, T)
    m.use_graph = graph
    m._offset_dev = torch.full((1,), base, dtype=torch.int64, device="cuda")
    m.rollout_infer_device(obs, idx, E, T, act, lp, val)
    assert int(m._offset_dev.cpu()[0]) == base + T
    return act.cpu().numpy(), lp.cpu().numpy(), val.cpu().numpy(), _pi_head(m, E)


def _launches(lib, m, obs, idx, E, T):
    act, lp, val = _outputs(m, E, T)
    m.use_graph = False
    m._offset_dev = torch.zeros(1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    n0 = lib.xtb_launch_count()
    m.rollout_infer_device(obs, idx, E, T, act, lp, val)
    torch.cuda.synchronize()
    return lib.xtb_launch_count() - n0


@pytest.fixture(params=[1, 0], ids=["fused", "layers"])
def fuse(request, xb):
    xb["lib"].xtb_set_fuse_heads(request.param)
    yield request.param
    xb["lib"].xtb_set_fuse_heads(1)


# (E, T) at max_batch 320: one step per chunk; several full chunks and a ragged one (E = 32 as in PPO C2, E = 37 not a
# multiple of 16, E = 150 beyond one 128-row tile, so the dense split-K is planned for two row tiles); E = 1 with
# T > max_batch, the most split-K partial sums a chunk can need
SHAPES = [(320, 2), (32, 23), (37, 19), (150, 5), (1, 700)]


@pytest.mark.parametrize("E,T", SHAPES, ids=["E%d_T%d" % s for s in SHAPES])
@pytest.mark.parametrize("kind", ["cnn", "impala", "mlp"])
def test_chunked_rollout_equals_single_steps(xb, tc_mode, fuse, kind, E, T):
    """a graph-replayed T-step call = T eager one-step calls on step t's rows from offset base + t, bit for bit; rows
    [0, E) of the pi head's tensor hold the last step's head afterwards"""
    m = _model(kind)
    obs, idx = _obs(kind, E, T, seed=E * 1000 + T)
    base = 1000
    act, lp, val, head = _infer(m, obs, idx, E, T, base, graph=True)
    for t in range(T):
        o_t, i_t = (obs, idx[t]) if idx is not None else (obs[t * E:(t + 1) * E], None)
        a1, l1, v1, h1 = _infer(m, o_t, i_t, E, 1, base + t, graph=False)
        assert np.array_equal(act[t], a1[0]), t
        assert np.array_equal(lp[t], l1[0]) and np.array_equal(val[t], v1[0]), t
    assert np.array_equal(head, h1)
    assert np.isfinite(lp).all() and np.isfinite(val).all()


@pytest.mark.parametrize("E", [32, 37, 150])
@pytest.mark.parametrize("kind", ["cnn", "mlp"])
def test_launches_per_chunk(xb, tc_mode, fuse, kind, E):
    """T = max_batch // E steps launch what one step does; one step more launches one more chunk"""
    m = _model(kind)
    c = MAX_BATCH // E
    obs, idx = _obs(kind, E, c + 1, seed=E)
    _launches(xb["lib"], m, obs, idx, E, 1)       # first call: any pending weight-blob refresh
    one = _launches(xb["lib"], m, obs, idx, E, 1)
    assert _launches(xb["lib"], m, obs, idx, E, c) == one
    assert _launches(xb["lib"], m, obs, idx, E, c + 1) == 2 * one - 1     # the counter bump runs once per call
