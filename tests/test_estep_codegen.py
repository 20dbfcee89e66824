"""Code-generation guard for the tensor E-step and the scoring kernel (no GPU needed): every instance of
estep_tc_kernel<D, NSG> and score_tc_kernel<D, NSG> compiles for sm_90a without register spills, and at D = 16 and 24
without a ptxas C75xx line (wgmma serialised or a compiler-inserted warpgroup wait/arrive).  Their software-pipelined MMA
sequence (tc_tile_logits) only overlaps MMAs with the epilogue while ptxas keeps the wgmma asynchronous; it still runs,
only slower, when it does not.  At D = 8 ptxas serialises the instances with one and two supergroups (C7520, as before
the pipelined schedule); the test keeps every other instance clean."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")
DIMS = (8, 16, 24)
NSGS = (1, 2, 3, 4)
KNOWN_SERIALISED = {("estep", 8, 1), ("estep", 8, 2), ("score", 8, 1), ("score", 8, 2)}


def test_estep_and_score_kernels_no_spills_no_serialisation(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "kernels_tc.o"), os.path.join(CSRC, "kernels_tc.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]

    def instance(name):
        m = re.search(r"(estep|score)_tc_kernelILi(\d+)ELi(\d+)E", name)
        return (m.group(1), int(m.group(2)), int(m.group(3))) if m else None

    perf, spill, current = {}, {}, None
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"\((C75\d\d)\).*function '([^']+)'", ln)
        if m and instance(m.group(2)):
            perf.setdefault(instance(m.group(2)), set()).add(m.group(1))
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = instance(m.group(1))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current:
            spill[current] = int(m.group(1)) + int(m.group(2))
            current = None
    expected = {(k, d, s) for k in ("estep", "score") for d in DIMS for s in NSGS}
    assert set(spill) == expected, sorted(spill)
    assert not {k: v for k, v in spill.items() if v}, spill
    assert not {k: v for k, v in perf.items() if k not in KNOWN_SERIALISED}, perf
