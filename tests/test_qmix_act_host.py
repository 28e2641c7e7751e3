"""CPU tier: acting for many QMIX / SCC environments in one call (QMixModel.act, QMixAlg.predict_with_selector_envs) on
the host side: the host-order uniforms and the inverse-CDF rule reproduce EpsilonGreedyActionSelector.select_action, the
arguments act refuses before anything reaches the device, and the kernels of csrc/agent_act.cuh compile for sm_90a
without register spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import qmix_act_oracle as qa

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which(NVCC) is not None


def _rows(rng, N, n, A):
    """Q values with exact ties and action weights with single-available rows and weights other than 0 / 1."""
    q = rng.normal(size=(N, n, A)).astype(np.float32)
    q[::3, :, 1:4] = q[::3, :, :1] + 0 * q[::3, :, 1:4]          # actions 0..3 tie
    q[1::4, 0, :] = 0.5                                           # a whole row ties
    avail = (rng.random((N, n, A)) < 0.6).astype(np.int32)
    avail[:, :, min(2, A - 1)] = 1                                # never an empty row
    avail[::5, 0, :] = 0
    avail[::5, 0, A - 1] = 1                                      # one available action, the last
    avail[2::5, 1 % n, :] = rng.integers(0, 4, size=(len(range(2, N, 5)), A))
    avail[2::5, 1 % n, 0] = 3                                     # weights 0..3
    return q, avail


@pytest.mark.parametrize("mode", ["annealing", "greedy", "random"])
@pytest.mark.parametrize("N,n,A", [(1, 2, 7), (9, 3, 5), (40, 8, 14), (7, 1, 3), (6, 2, 1)])
def test_selector_uniforms_reproduce_the_host_selector(mode, N, n, A):
    from xingtian_b200.algorithm.qmix import EpsilonGreedyActionSelector, QMixAlg
    start = {"annealing": 1.0, "greedy": 1.0, "random": 1.0}[mode]
    finish = {"annealing": 0.05, "greedy": 0.05, "random": 1.0}[mode]
    sel = EpsilonGreedyActionSelector(dict(epsilon_start=start, epsilon_finish=finish, epsilon_anneal_time=100))
    rng = np.random.default_rng(N * 100 + n * 10 + A)
    q, avail = _rows(rng, N, n, A)
    test_mode = mode == "greedy"
    t_env = 40
    np.random.seed(123)
    want = np.concatenate([sel.select_action(q[e:e + 1], avail[e:e + 1], t_env, test_mode=test_mode) for e in range(N)])
    after = np.random.rand()
    eps = np.full(N, sel.epsilon)
    assert eps[0] == {"annealing": 1.0 - 0.95 * 40 / 100, "greedy": 0.0, "random": 1.0}[mode]
    np.random.seed(123)
    u = QMixAlg.selector_uniforms(N, n)
    assert np.random.rand() == after        # the same numbers of the stream, no more and no fewer
    got = qa.select_actions(q, avail, eps, u)
    assert np.array_equal(got, want)
    if mode != "annealing":
        assert np.all((u[:, 0] < eps[:, None]) == (mode == "random"))


def test_uniforms_are_the_host_draw_order():
    from xingtian_b200.algorithm.qmix import QMixAlg
    np.random.seed(5)
    u = QMixAlg.selector_uniforms(3, 4)
    np.random.seed(5)
    assert np.array_equal(u, np.random.rand(3, 2, 4))


class _Stub(object):
    """QMixModel's acting checks without a device: the attributes act reads before anything is staged."""

    def __init__(self, n=2, A=5, o=4, act_envs=3, last=True, ident=True):
        from xingtian_b200.model.qmix import QMixModel
        m = QMixModel.__new__(QMixModel)
        m.n_agents, m.n_actions, m.act_envs, m.obs_last_action, m.obs_agent_id = n, A, act_envs, last, ident
        m.obs_shape = o + (A if last else 0) + (n if ident else 0)
        self.m = m


def test_act_rejects_bad_arguments_on_the_host():
    m = _Stub().m
    assert m.act_obs_dim == 4
    obs = np.zeros((2, 2, 4), np.float32)
    avail = np.ones((2, 2, 5), np.int32)
    reset = np.zeros(2, bool)
    bad = [dict(obs=np.zeros((2, 2, 11))),                             # the assembled width, not the raw one
           dict(obs=np.zeros((2, 4))),
           dict(obs=np.zeros((4, 2, 4)), avail=np.ones((4, 2, 5), np.int32), reset=np.zeros(4)),   # 4 > act_envs
           dict(avail=np.ones((2, 2, 5), np.float32)),                 # weights are integers
           dict(avail=np.ones((2, 2, 4), np.int32)),
           dict(avail=np.where(np.arange(5) == 1, -1, 1) * np.ones((2, 2, 1), np.int32)),   # a negative weight
           dict(avail=np.concatenate([np.ones((1, 2, 5)), np.zeros((1, 2, 5))]).astype(np.int32)),   # an empty row
           dict(reset=np.zeros(3)),
           dict(uniforms=np.zeros((2, 2, 3))),
           dict(epsilon=np.zeros(3))]
    for over in bad:
        args = dict(obs=obs, avail=avail, reset=reset, epsilon=0.1, uniforms=None)
        args.update(over)
        with pytest.raises(ValueError):
            m.act(**args)
    m2 = _Stub(last=False, ident=False).m
    assert m2.act_obs_dim == m2.obs_shape == 4


def test_model_config_rejects_no_environments():
    from xingtian_b200.model.qmix import QMixModel
    m = QMixModel.__new__(QMixModel)
    with pytest.raises(ValueError, match="act_envs"):
        m._agent_config(dict(model_config=dict(n_agents=2, obs_shape=4, rnn_hidden_dim=8, episode_limit=4, n_actions=3, batch_size=2,
                                               state_shape=[3], act_envs=0)))


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_agent_act_kernels_do_not_spill(repo_root, tmp_path):
    csrc = os.path.join(repo_root, "xingtian_b200", "csrc")
    src = tmp_path / "agent_act_only.cu"
    src.write_text('#include "{0}/agent_act.cuh"\n'.format(csrc))
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o",
           str(tmp_path / "a.cubin"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    kernels, cur = {}, None
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1) if "agent_act" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = tuple(int(x) for x in m.groups())
    assert len(kernels) == 2, sorted(kernels)
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
