"""Code-generation guard for the tensor M-step (no GPU needed): every instantiation of
mstep_tc_kernel must compile for sm_90a with its warpgroup MMAs left asynchronous and
without register spills.  ptxas reports a serialised wgmma pipeline only as an info
line (C75xx "wgmma ... serialized"), and the kernel still runs, only slower; this
test turns that line into a failure."""
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")
MSTEP_DIMS = (4, 8, 12, 16, 20, 24)


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_mstep_wgmma_not_serialised_and_no_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "kernels_tc.o"), os.path.join(CSRC, "kernels_tc.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    log = res.stdout + res.stderr

    serialised = [ln for ln in log.splitlines()
                  if "mstep_tc_kernel" in ln and re.search(r"wgmma.*serializ|C75\d\d", ln)]
    assert not serialised, "\n".join(serialised)

    # ptxas prints "Compiling entry function '<name>'" and then the function's properties
    spills, seen = {}, set()
    current = None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current and "mstep_tc_kernel" in current:
            d = int(re.search(r"mstep_tc_kernelILi(\d+)E", current).group(1))
            seen.add(d)
            if int(m.group(1)) or int(m.group(2)):
                spills[d] = ln.strip()
            current = None
    assert seen == set(MSTEP_DIMS), sorted(seen)
    assert not spills, spills
