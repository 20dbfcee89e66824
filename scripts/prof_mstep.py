"""Where the tensor M-step's time goes: the M-step alone (mstep_tc_kernel + mstep_tc_finalize_kernel) at config 3
(N = 10M, D = 24, K = 64) and config 2 (N = 1M, D = 16, K = 32), for one or more builds of the library, each timed in a
process of its own (GMM_B200_LIB).

The timing variants are built from kernels_tc.cu with GMM_MSTEP_CUT (the default build is 0):
    make -C cuda-gmm-mpi_b200/csrc variant NAME=mcut1 DEFS=-DGMM_MSTEP_CUT=1   # operand build and loads only: no MMAs
    make -C cuda-gmm-mpi_b200/csrc variant NAME=mcut2 DEFS=-DGMM_MSTEP_CUT=2   # MMAs on unsplit data: no feature build
    make -C cuda-gmm-mpi_b200/csrc variant NAME=mcut3 DEFS=-DGMM_MSTEP_CUT=3   # no drains of the accumulators
then
    python scripts/prof_mstep.py [--launches 40] default cuda-gmm-mpi_b200/variants/libgmm_b200_mcut1.so ...
(the results of a cut variant are wrong; only its time means something).

Per library and shape: one E-step for the responsibilities, 3 warm-up M-steps, then the CUDA-event time of `--launches`
M-steps (the engine's per-phase timer brackets the two kernels); the median of 3 such blocks is printed as ms per launch.
Beside it, two times computed from the shapes (not measured):
  - the tensor floor: the executed MMAs at 4096 FP16 flop per clock and SM, at the card's maximum SM clock;
  - the shared-memory model at 128 bytes per clock and SM: the bytes every 32-event sub-tile of a CTA moves through shared
    memory, times the sub-tiles an SM runs, for the staged feature operand of earlier builds and for the register feature
    operand in the schedule launch_mstep_d() picks for K (32 clusters per CTA at K <= 32; at K > 32 two CTAs per event
    range, each with half of the feature rows and 64 clusters).
The number of warpgroup MMA instructions (HGMMA) in each library's mstep_tc_kernel is counted with cuobjdump -sass, so
a variant whose MMAs the compiler dropped is visible.  The card's name, power limit and maximum SM clock are printed
first.  Needs a GPU; the M-step runs on the tensor path only (no SIMT fall-back).
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
KTE = 32


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:                       # noqa: BLE001
        return f"unknown ({e})"


def tiles(D):
    """Feature tiles (MT) of MCfg<D> and the rows the staged path builds (NCHUNK * 8)."""
    S = D // 4
    rpp = 1 + 2 * S + S * (D // 2)
    rows = 4 * ((rpp + 7) // 8) * 8
    return (rows + 127) // 128, rows


def ncl(K, register_a=True):
    """Clusters per CTA of launch_mstep_d() (the staged path always had 32)."""
    return 64 if register_a and K > 32 else 32


def subtiles_per_sm(N, K, sms, register_a=True):
    """launch_mstep_d(): contiguous event ranges of whole sub-tiles, NCL / 32 CTAs per range and NCL clusters; an SM runs
    ceil(CTAs / SMs) CTAs one after the other."""
    per = -(-N // sms)
    per = -(-per // KTE) * KTE
    gx = -(-N // per)
    c = ncl(K, register_a)
    gy = -(-K // c)
    return -(-(gx * (c // 32) * gy) // sms) * (per // KTE)


def smem_bytes_per_subtile(D, K, register_a):
    """Shared-memory bytes one 32-event sub-tile of a CTA moves, per operand path."""
    mt, rows = tiles(D)
    nct = 128 * mt
    c = ncl(K, register_a)
    hpc = 64 // c                                     # 64-row halves per consumer warpgroup
    b = mt * hpc * 2 * 3 * c * 16 * 2                 # wgmma B reads: per consumer, half and k-step gh, gl, gs (c * 32 B each)
    gam = c * KTE * 4 + 3 * c * KTE * 2 + D * KTE * 4 + c * KTE * 4   # raw gamma read, images written, TMA writes
    drains = nct * 32 * 4 * 2 // 4 + nct * 32 * 4 * 2 // 16    # racc read + write: exact group every 4, remainder every 16
    if register_a:
        a = nct * (1 + 2 * hpc) * 8 * 4               # each consumer thread: 1 + 2 per half dimensions x 8 events of z
    else:
        a = rows * KTE * 2 * 2                        # builders write ph / pl
        a += mt * 2 * 2 * 3 * 64 * 16 * 2             # wgmma A reads: per half and k-step ah twice, al once (2 KB each)
        a += 4 * D * KTE * 4                          # builders read the z tile
    return a + b + gam + drains


def mma_flops_per_subtile(D, K):
    mt, _ = tiles(D)
    c = ncl(K)
    return mt * (64 // c) * 2 * 3 * 64 * c * 16 * 2  # per consumer warpgroup: halves x 2 k-steps x 3 m64n{c}k16


def hgmma_count(lib, D, K):
    """HGMMA instructions in the mstep_tc_kernel<D, NCL> that runs at K (any NCL in a library that has one template argument),
    from cuobjdump -sass, or None when cuobjdump is missing."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        return None
    out = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    count, inside = 0, False
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            inside = re.search(rf"mstep_tc_kernelILi{D}E(Li{ncl(K)}E)?E", m.group(1)) is not None
            continue
        if inside and "HGMMA" in ln and "gdesc[URZ]" not in ln:     # (ptxas's empty HGMMA of a lone commit does no work)
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
        eng.estep(K)
        for _ in range(3):
            eng.mstep(K)
        blocks = []
        for _ in range(3):
            eng.profile(reset=True)
            for _ in range(launches):
                eng.mstep(K)
            p = eng.profile(reset=True)
            blocks.append(p["mstep_ms"] / launches)
    return dict(shape=shape, N=N, D=D, K=K, mstep_ms=round(float(np.median(blocks)), 4), tensor_launches=p["mstep_tensor_launches"],
                blocks_ms=[round(b, 4) for b in blocks], sm_clock_after=smi("clocks.sm"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*", default=["default"], help="library paths, or 'default' for the in-tree build")
    ap.add_argument("--launches", type=int, default=40)
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
    for shape in a.shapes.split(","):
        N, D, K = SHAPES[shape]
        n_sub = subtiles_per_sm(N, K, sms)
        n_sub_staged = subtiles_per_sm(N, K, sms, register_a=False)
        clk = max_mhz * 1e3                           # clocks per ms
        model = dict(
            clusters_per_cta=ncl(K),
            tensor_floor_ms=round(n_sub * mma_flops_per_subtile(D, K) / 4096 / clk, 4),
            smem_model_staged_ms=round(n_sub_staged * smem_bytes_per_subtile(D, K, False) / 128 / clk, 4),
            smem_model_register_a_ms=round(n_sub * smem_bytes_per_subtile(D, K, True) / 128 / clk, 4),
            smem_bytes_per_subtile=dict(staged=smem_bytes_per_subtile(D, K, False), register_a=smem_bytes_per_subtile(D, K, True)))
        print(json.dumps(dict(shape=shape, subtiles_per_sm=n_sub, **model)), flush=True)
        for lib in a.libs:
            env = dict(os.environ)
            path = os.path.join(ROOT, "cuda-gmm-mpi_b200", "libgmm_b200.so") if lib == "default" else os.path.abspath(lib)
            if lib != "default":
                env["GMM_B200_LIB"] = path
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", shape, "--launches", str(a.launches)], env=env,
                               capture_output=True, text=True, timeout=1200)
            lines = r.stdout.strip().splitlines()
            if r.returncode != 0 or not lines:
                print(json.dumps(dict(shape=shape, lib=os.path.basename(lib), error=r.stderr[-800:])), flush=True)
                continue
            res = json.loads(lines[-1])
            res["lib"] = os.path.basename(lib)
            res["hgmma_in_kernel"] = hgmma_count(path, D, K)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
