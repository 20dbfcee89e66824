"""Row layout of the tensor M-step's feature operand (csrc/mstep_rows.h), at every compiled D, without a GPU.

The layout is compiled on the host with the system C++ compiler and printed.  Checked:
  * every packed statistic comes from exactly one operand row, and each row's factors multiply to that statistic
    (z_i z_j, z_i * 1, or 1 * 1);
  * each statistic stays in the feature tile of the earlier layout (test_mstep_error_model.feature_tiles), so the chain
    stagger of its FP32 partial sums is unchanged;
  * the four rows of a consumer thread share their first factor: at most 5 rows of the z tile per thread and sub-tile;
  * the shared-memory wavefronts of the z loads: for an 8-event (32-byte) load of one factor by the 8 lane groups of a
    warp, rows of the SWIZZLE_128B tile in bank group (row >> 1) & 3 share 8 banks, so a load takes as many wavefronts
    as the most distinct rows in one bank group (2 is the least for 8 distinct rows, 8 the unswizzled tile's worst).
The numbers are printed with -s (pytest -s tests/test_mstep_rowmap.py)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from test_mstep_error_model import feature_tiles

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")
MSTEP_DIMS = (4, 8, 12, 16, 20, 24)
ONE = 32

DRIVER = r"""
#include <cstdio>
#include "mstep_rows.h"
int main() {
    for (int D : {4, 8, 12, 16, 20, 24}) {
        const std::vector<gmm::MRow> rows = gmm::mstep_row_layout(D);
        std::printf("D %d %d\n", D, (int)rows.size());
        for (const gmm::MRow& r : rows) std::printf("%d %d %d %d %d\n", r.f, r.i, r.j, r.a, r.b);
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def layouts(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("rowmap")
    src, exe = d / "rows.cpp", d / "rows"
    src.write_text(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, "-o", str(exe), str(src)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    res, k = {}, 0
    while k < len(out) and out[k]:
        _, D, n = out[k].split()
        D, n = int(D), int(n)
        res[D] = np.array([[int(v) for v in ln.split()] for ln in out[k + 1:k + 1 + n]], np.int64).reshape(n, 5)
        k += 1 + n
    return res


def thread_rows(mt, w, gid):
    """Operand rows of consumer thread (warp w of tile mt's warpgroup, lane group gid), slot order 2 h + s."""
    return [mt * 128 + h * 64 + w * 16 + gid + 8 * s for h in (0, 1) for s in (0, 1)]


def waves(codes):
    rows = set(int(c) for c in codes)
    cnt = [0, 0, 0, 0]
    for r in rows:
        cnt[((r if r < ONE else r - ONE) >> 1) & 3] += 1
    return max(cnt)


@pytest.mark.parametrize("D", MSTEP_DIMS)
def test_rowmap_covers_each_statistic_once_in_its_tile(layouts, D):
    L = layouts[D]
    F = 1 + D + D * (D + 1) // 2
    S = D // 4
    assert len(L) == 128 * ((4 * ((1 + 2 * S + S * (D // 2) + 7) // 8) * 8 + 127) // 128)
    used = L[L[:, 0] >= 0]
    assert sorted(used[:, 0].tolist()) == list(range(F))
    tile = feature_tiles(D)
    rows = np.nonzero(L[:, 0] >= 0)[0]
    assert (rows // 128 == tile[L[rows, 0]]).all()
    for f, i, j, a, b in used:
        fa = [x for x in (a, b) if x < ONE]
        if f == 0:
            assert fa == [] and i < 0 and j < 0
        elif f <= D:
            assert fa == [f - 1] and i == f - 1 and j < 0
        else:
            assert sorted(fa) == sorted([i, j]) and f == 1 + D + i * (i + 1) // 2 + j and 0 <= j <= i < D
    assert ((L[:, 3] < D) | (L[:, 3] >= ONE)).all() and ((L[:, 4] < D) | (L[:, 4] >= ONE)).all()
    assert (L[:, 3] < ONE + 8).all() and (L[:, 4] < ONE + 8).all()


@pytest.mark.parametrize("D", MSTEP_DIMS)
def test_rowmap_loads_per_thread_and_bank_groups(layouts, D):
    L = layouts[D]
    MT = len(L) // 128
    dims, wa, wb = [], [], []
    for mt in range(MT):
        for w in range(4):
            a_codes, b_codes = [], [[] for _ in range(4)]
            for gid in range(8):
                r = thread_rows(mt, w, gid)
                assert len(set(L[r, 3].tolist())) == 1, "the rows of a thread share their first factor"
                a_codes.append(L[r[0], 3])
                dims.append(len({x for x in L[r, 3].tolist() + L[r, 4].tolist() if x < ONE}))
                for s in range(4):
                    b_codes[s].append(L[r[s], 4])
            wa.append(waves(a_codes))
            wb += [waves(c) for c in b_codes]
    assert max(dims) <= 5
    assert max(wa) <= 3 and max(wb) <= 4
    print(f"D={D}: distinct dimensions per thread <= {max(dims)}; wavefronts per 8-event load: shared factor "
          f"max {max(wa)}, other factors max {max(wb)}, mean {np.mean(wa + wb):.2f} (8-way without the swizzle)")
