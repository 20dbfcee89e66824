"""Code-generation guard for gmm_condition (no GPU needed): every instance of condition_simt_kernel (observed and imputed
counts rounded up to multiples of 4, 36 instances for D <= 32) is built for sm_90a without a register spill or other
local memory."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")


def test_condition_kernels_built_without_local_memory(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I/usr/include", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "gmm_api.o"), os.path.join(CSRC, "gmm_api.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, frames = None, {}
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1) if "condition_simt_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current:
            frames[current] = sum(int(v) for v in m.groups())
            current = None
    assert len(frames) == 36, sorted(frames)
    bad = {n: s for n, s in frames.items() if s}
    assert not bad, bad
