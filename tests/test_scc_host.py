"""CPU tier: the SCC kernels (scc.cuh) compile for sm_90a without register spills, and SCCAlg hands SCCModel.train
exactly what the reference's QMixAlg hands QMixModel.train (tests/golden/qmix.npz), with the raw observations second."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import qmix_alg_scenario as sc

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which(NVCC) is not None
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qmix.npz")


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_scc_kernels_do_not_spill(repo_root, tmp_path):
    csrc = os.path.join(repo_root, "xingtian_b200", "csrc")
    src = tmp_path / "scc_only.cu"
    src.write_text('#include "{0}/gemm_f32.cuh"\n#include "{0}/scc.cuh"\n'.format(csrc))
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o",
           str(tmp_path / "s.cubin"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    kernels, cur = {}, None
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1) if "scc" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = tuple(int(x) for x in m.groups())
    assert len(kernels) == 6, sorted(kernels)
    assert all(v[1:] == (0, 0) for v in kernels.values()), kernels


def test_scc_alg_passes_the_raw_observations_second():
    from xingtian_b200.algorithm.qmix import EpisodeBatch
    from xingtian_b200.algorithm.scc import SCCAlg
    from xingtian_b200.registry import Registers

    class SccRecordingModel(sc.RecordingActor):
        pass

    Registers.model(SccRecordingModel)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "SccRecordingModel"
    alg = SCCAlg(model_info, alg_config)
    assert alg.alg_name == "SCCAlg"
    out = sc.drive(alg, lambda a: EpisodeBatch(a.scheme, a.groups, 1, sc.LIMIT + 1, preprocess=a.preprocess))
    with np.load(GOLDEN) as g:
        gold = {k: g[k] for k in g.files}
    names = ("trajectories", "obs_len", "avail", "actions", "cur_stats", "target_stats", "rewards", "terminated", "mask")
    assert len(alg.actor.trained) == int(gold["n_trained"])
    for k, args in enumerate(alg.actor.trained):
        assert len(args) == 10
        obs = args[1]
        assert obs.shape == (4, sc.LIMIT + 1, sc.N_AGENTS, sc.OBS)
        np.testing.assert_array_equal(obs, args[0][..., :sc.OBS])
        for name, a in zip(names, args[:1] + args[2:]):
            assert np.array_equal(a, gold["train%d_%s" % (k, name)]), (k, name)
    for key in ("acted", "epsilon", "synced_after_train"):
        assert np.array_equal(out[key], gold[key]), key
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "SccRecordingModel"
    idle = SCCAlg(model_info, alg_config)
    with pytest.raises(KeyError, match="scc need to dist dummy model"):
        idle.train_ready(0)
    assert np.isnan(idle.train(episode_num=1))
