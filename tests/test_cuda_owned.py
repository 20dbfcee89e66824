"""Ownership of the engine's CUDA allocations, events and streams (csrc/cuda_owned.h).

Every device or pinned buffer, event and stream of the engine is held by an owner that frees it, and lazy buffers grow
through reserve(), which leaves an array empty and the runtime's last error clear when an allocation fails.  Checked here:
no source outside the header allocates or frees by hand; a host program built from the header exercises reserve() with
and without a device; and gmm_seed_kmeans sizes its cross-rank transfer buffers from the communicator of each call."""
import os
import re
import subprocess
import threading

import numpy as np
import pytest

from conftest import ROOT, gpu_count
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")
RAW_CALL = re.compile(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(")


def test_no_raw_allocation_outside_the_owners():
    hits = []
    for base, _, files in os.walk(CSRC):
        for name in sorted(files):
            if name == "cuda_owned.h" or not name.endswith((".cu", ".cuh", ".h", ".cpp")):
                continue
            path = os.path.join(base, name)
            with open(path, encoding="utf-8") as f:
                for i, line in enumerate(f, 1):
                    if RAW_CALL.search(line):
                        hits.append(f"{os.path.relpath(path, CSRC)}:{i}: {line.strip()}")
    assert not hits, "allocate, free, create or destroy through csrc/cuda_owned.h:\n" + "\n".join(hits)


_PROGRAM = r"""
#include <cstdio>
#include <utility>
#include "cuda_owned.h"
using namespace gmm;

#define CHECK(cond) do { if (!(cond)) { std::printf("FAILED line %d: %s\n", __LINE__, #cond); return 1; } } while (0)

// A request no allocator can serve fails at once and leaves the array empty.  With a device, the runtime's last error is
// clear afterwards; without a driver the runtime reports its failed initialisation on every call, cleared or not.
template <typename A> static int huge_request_fails(bool device) {
    A a;
    CHECK(a.reserve((size_t)1 << 62) == GMM_ERR_CUDA);
    CHECK(a.get() == nullptr && a.size() == 0);
    CHECK(!device || cudaGetLastError() == cudaSuccess);
    return 0;
}

int main() {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess) ndev = 0;
    const bool device = ndev > 0;
    if (huge_request_fails<DeviceArray<char>>(device) || huge_request_fails<PinnedArray<char>>(device) ||
        huge_request_fails<DeviceArray<double>>(device) || huge_request_fails<PinnedArray<double>>(device))
        return 1;
    DeviceArray<float> a;
    if (ndev > 0) {
        CHECK(a.reserve(1000) == GMM_OK && a.get() != nullptr && a.size() == 1000);
        float* p = a;
        CHECK(a.reserve(10) == GMM_OK && a.get() == p && a.size() == 1000);
        CHECK(a.reserve(4000) == GMM_OK && a.get() != nullptr && a.size() == 4000);
        CHECK(cudaMemset(a, 0, sizeof(float) * a.size()) == cudaSuccess);
        PinnedArray<double> h;
        CHECK(h.reserve(16) == GMM_OK && h.size() == 16);
        h[15] = 1.0;
        h.reset();
        CHECK(h.get() == nullptr && h.size() == 0);
        Event e;
        CHECK(e.create(cudaEventDisableTiming) == GMM_OK && (cudaEvent_t)e != nullptr);
        cudaEvent_t first = e;
        CHECK(e.create(cudaEventDisableTiming) == GMM_OK && (cudaEvent_t)e == first);
        Stream s;
        CHECK(s.create(cudaStreamNonBlocking) == GMM_OK && (cudaStream_t)s != nullptr);
        CHECK(cudaEventRecord(e, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess);
    }
    const size_t held = a.size();
    float* const p = a;
    DeviceArray<float> b(std::move(a));
    CHECK(a.get() == nullptr && a.size() == 0);
    CHECK(b.get() == p && b.size() == held);
    DeviceArray<float> c;
    c = std::move(b);
    CHECK(b.get() == nullptr && b.size() == 0 && c.get() == p && c.size() == held);
    c.reset();
    CHECK(c.get() == nullptr && c.size() == 0);
    CHECK(!device || cudaGetLastError() == cudaSuccess);
    std::printf("ok devices=%d\n", ndev);
    return 0;
}
"""


def test_reserve_and_handles(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "owned_check.cu"
    src.write_text(_PROGRAM)
    exe = tmp_path / "owned_check"
    subprocess.run([nvcc, "-std=c++17", "-I", CSRC, "-o", str(exe), str(src), os.path.join(CSRC, "host_math.cpp"),
                    "-Xcompiler", "-fopenmp", "-lgomp"], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr


@pytest.mark.gpu
def test_seed_kmeans_before_and_after_comm_init():
    """k-means++ run once on each shard alone, then again over the communicator, chooses what a fresh sharded run chooses:
    the transfer buffers of the first call (one rank) grow to the ranks of the second.  max_iter = 0 keeps the centres to
    the k-means++ picks, which do not depend on the moments the first call fixed from its own shard."""
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import __graft_entry__ as entry
    pkg = entry.load_package()
    pkg.load_library()
    G, N, D, K = 2, 60_001, 16, 24
    x = pkg.synth.make_blobs(N, D, 12, seed=1051)

    def run(early):
        uid = pkg.nccl_unique_id()
        out, errs = [None] * G, [None] * G

        def worker(g):
            try:
                b, n = pkg.shard_range(N, G, g)
                with pkg.Engine(np.ascontiguousarray(x[b:b + n]), K, device=g, n_global=N, offset=b) as eng:
                    if early:
                        eng.seed_kmeans(K, max_iter=0, seed=5)
                    eng.comm_init(G, g, uid)
                    out[g] = eng.seed_kmeans(K, max_iter=0, seed=5)
            except Exception as ex:  # noqa: BLE001
                errs[g] = ex

        ts = [threading.Thread(target=worker, args=(g,)) for g in range(G)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=600)
        for g in range(G):
            assert errs[g] is None, f"rank {g}: {errs[g]}"
            assert out[g] is not None, f"rank {g} did not finish"
        return out

    fresh, again = run(False), run(True)
    for g in range(G):
        np.testing.assert_array_equal(again[g][1], fresh[g][1])
        assert again[g][3] == fresh[g][3]
