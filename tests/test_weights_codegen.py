"""Code-generation guard for the weighted instances of the tensor kernels (gmm_set_weights; no GPU needed): every
estep_tc_kernel<D, NSG, true> and mstep_tc_kernel<D, NCL, true> compiles for sm_90a without register spills, and without
a ptxas C75xx line (wgmma serialised) beyond the one the unweighted E-step already has at D = 8 with one or two
supergroups (tests/test_estep_codegen.py).  The weights add a load and a multiply to the M-step's responsibility warps,
whose register pool is 56 at three feature tiles, and a load to the E-step's log-likelihood."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")
KNOWN_SERIALISED = {("estep", 8, 1), ("estep", 8, 2)}


def test_weighted_tc_kernels_no_spills_no_serialisation(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "kernels_tc.o"), os.path.join(CSRC, "kernels_tc.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]

    def instance(name):
        m = re.search(r"(estep|mstep)_tc_kernelILi(\d+)ELi(\d+)ELb1E", name)
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
    expected = ({("estep", d, s) for d in (8, 16, 24) for s in (1, 2, 3, 4)} |
                {("mstep", d, ncl) for d in (4, 8, 12, 16, 20, 24) for ncl in (32, 64)})
    assert set(spill) == expected, sorted(spill)
    assert not {k: v for k, v in spill.items() if v}, spill
    assert not {k: v for k, v in perf.items() if k not in KNOWN_SERIALISED}, perf
