"""CPU tier: the QMIX kernels (qmix.cuh) compile for sm_90a without register spills (nvcc cross-compiles, no GPU)."""
import os
import re
import shutil
import subprocess

import pytest

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which(NVCC) is not None


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_qmix_kernels_do_not_spill(repo_root, tmp_path):
    csrc = os.path.join(repo_root, "xingtian_b200", "csrc")
    src = tmp_path / "qmix_only.cu"
    src.write_text('#include "{0}/gemm_f32.cuh"\n#include "{0}/qmix.cuh"\n'.format(csrc))
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o",
           str(tmp_path / "q.cubin"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    kernels, cur = {}, None
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1) if "qmix" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = tuple(int(x) for x in m.groups())
    assert len(kernels) == 5, sorted(kernels)
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
