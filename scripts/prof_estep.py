"""Where the tensor E-step's time goes: the E-step kernel alone at config 3 (N = 10M, D = 24, K = 64) and config 2
(N = 1M, D = 16, K = 32), for one or more builds of the library, each timed in a process of its own (GMM_B200_LIB).

The timing variants are built from kernels_tc.cu with GMM_ESTEP_CUT (the default build is 0):
    make -C cuda-gmm-mpi_b200/csrc variant NAME=mma DEFS=-DGMM_ESTEP_CUT=1       # MMA only: no squares, exp, log or stores
    make -C cuda-gmm-mpi_b200/csrc variant NAME=nostore DEFS=-DGMM_ESTEP_CUT=2   # full epilogue, responsibilities not written
then
    python scripts/prof_estep.py [--launches 50] default cuda-gmm-mpi_b200/variants/libgmm_b200_mma.so ...

Per library and shape: the parameters of the seed (valid whatever the variant computes: the E-step alone is timed, no
M-step runs), 5 warm-up launches, then the CUDA-event time of `--launches` E-step launches (the engine's per-phase timer
brackets the kernel launches only); the median of 3 such blocks is printed as ms per launch, with the tensor floor of the
MMAs at the card's maximum SM clock for comparison and the measured fraction of that floor.  The card's name, power limit,
maximum SM clock and the SM clock read right after the timed blocks are printed first.  Needs a GPU; the E-step runs on the
tensor path only (no SIMT fall-back).

A variant is only a valid cut when it issues every MMA of the full build: the compiler may drop the MMAs whose results a
variant no longer uses.  Each library's `HGMMA` count over the estep_tc_kernel instances (`cuobjdump -sass`) is printed
and a library whose count differs from the in-tree build's is flagged `"valid": false`.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as entry  # noqa: E402

SHAPES = {"c3": (10_000_000, 24, 64), "c2": (1_000_000, 16, 32)}


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:                       # noqa: BLE001
        return f"unknown ({e})"


def mma_cycles_per_sm(N, D, K, sms):
    """MMA issue cycles per SM if every m64nNk16 wgmma of a 64-event tile took N / 2 cycles (4096 FP16 flop per cycle
    and SM): per supergroup of 16 clusters and block c the k-steps (CP - c) + ceil((CP - c + 1) / 2), N = 128 columns."""
    cp = D // 8
    ksteps = sum((cp - c) + (cp - c + 2) // 2 for c in range(cp)) * ((K + 15) // 16)
    tiles = (N + 63) // 64
    return tiles * ksteps * 64 / sms


def lib_path(lib):
    return os.path.join(ROOT, "cuda-gmm-mpi_b200", "libgmm_b200.so") if lib == "default" else os.path.abspath(lib)


def estep_hgmma(path):
    """HGMMA instructions in the SASS of the library's estep_tc_kernel instances (None when cuobjdump is not found)."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        return None
    sass = subprocess.run([tool, "-sass", path], capture_output=True, text=True, timeout=600).stdout
    count, inside = 0, False
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            inside = "estep_tc_kernel" in m.group(1)
        elif inside and re.search(r"\bHGMMA\.", ln):
            count += 1
    return count


def run_one(shape, launches):
    pkg = entry.load_package()
    pkg.load_library()
    N, D, K = SHAPES[shape]
    ev = pkg.synth.make_blobs(N, D, K)
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", pkg.PATH_TENSOR)
        eng.seed(K)
        for _ in range(5):
            eng.estep(K)
        blocks = []
        for _ in range(3):
            eng.profile(reset=True)
            for _ in range(launches):
                eng.estep(K)
            blocks.append(eng.profile(reset=True)["estep_ms"] / launches)
    clock = smi("clocks.sm")
    return dict(shape=shape, N=N, D=D, K=K, estep_ms=round(float(np.median(blocks)), 4),
                blocks_ms=[round(b, 4) for b in blocks], sm_clock_after=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*", default=["default"], help="library paths, or 'default' for the in-tree build")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--shapes", default="c3,c2")
    ap.add_argument("--one", default=None, help=argparse.SUPPRESS)       # child: time one shape with GMM_B200_LIB
    a = ap.parse_args()
    if a.one:
        print(json.dumps(run_one(a.one, a.launches)), flush=True)
        return
    import torch
    print("card:", smi("name,power.limit,clocks.max.sm"), flush=True)
    try:
        max_mhz = float(smi("clocks.max.sm").split()[0])
    except ValueError:
        max_mhz = float("nan")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    full = estep_hgmma(lib_path("default"))
    hgmma = {lib: estep_hgmma(lib_path(lib)) for lib in a.libs}
    for lib in a.libs:
        print(json.dumps(dict(lib=os.path.basename(lib), estep_hgmma=hgmma[lib], in_tree_hgmma=full,
                              valid=hgmma[lib] is not None and hgmma[lib] == full)), flush=True)
    for shape in a.shapes.split(","):
        N, D, K = SHAPES[shape]
        floor = mma_cycles_per_sm(N, D, K, sms) / (max_mhz * 1e3)
        for lib in a.libs:
            env = dict(os.environ)
            if lib != "default":
                env["GMM_B200_LIB"] = lib_path(lib)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", shape, "--launches", str(a.launches)], env=env,
                               capture_output=True, text=True, timeout=1200)
            lines = r.stdout.strip().splitlines()
            if r.returncode != 0 or not lines:
                print(json.dumps(dict(shape=shape, lib=os.path.basename(lib), error=r.stderr[-800:])), flush=True)
                continue
            res = json.loads(lines[-1])
            res["lib"] = os.path.basename(lib)
            res["mma_floor_ms_at_max_clock"] = round(floor, 4)
            res["floor_fraction"] = round(floor / res["estep_ms"], 3)
            res["valid"] = hgmma[lib] is not None and hgmma[lib] == full
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
