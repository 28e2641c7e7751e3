"""CPU tier: what ptxas makes of the wgmma GEMM kernels (no GPU needed, nvcc cross-compiles for sm_90a).

A branch or trip count that ptxas cannot prove warp-uniform inside a wgmma issue loop, or a register write to an
accumulator while wgmma groups are in flight, makes ptxas serialize every wgmma of the kernel (C7520 / C7515): the
code stays correct and only gets slower, so nothing else would notice."""
import os
import re
import shutil
import subprocess

import pytest

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which(NVCC) is not None


@pytest.fixture(scope="module")
def ptxas_log(repo_root, tmp_path_factory):
    src = os.path.join(repo_root, "xingtian_b200", "csrc", "xtb_engine.cu")
    out = str(tmp_path_factory.mktemp("ptxas") / "xtb_engine.cubin")
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o", out, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return res.stdout + res.stderr


def gemm_kernels(log):
    """{mangled name: (registers, stack bytes, spill store bytes, spill load bytes)} of bp_rows_kernel / bp_wgrad_kernel."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1) if re.search(r"bp_(rows|wgrad)_kernel", m.group(1)) else None
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            out.setdefault(cur, [None, 0, 0, 0])[1:] = [int(x) for x in m.groups()]
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out.setdefault(cur, [None, 0, 0, 0])[0] = int(m.group(1))
    return out


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_wgmma_issue_is_not_serialized(ptxas_log):
    serialized = sorted(set(re.findall(r"\((C75\d\d)\) Potential Performance Loss: wgmma[^']*'([^']+)'", ptxas_log)))
    assert not serialized, serialized
    assert "C7520" not in ptxas_log


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_gemm_kernels_do_not_spill(ptxas_log):
    kernels = gemm_kernels(ptxas_log)
    assert len(kernels) == 16, sorted(kernels)          # bp_rows_kernel<KIND 0..2, N 16..64>, bp_wgrad_kernel<N 16..64>
    spilling = {k: v for k, v in kernels.items() if v[1] or v[2] or v[3]}
    assert not spilling, spilling
