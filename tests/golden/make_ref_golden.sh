#!/bin/bash
# Generates tests/golden/ref_c1.* and ref_c1_it20.* by running the UNMODIFIED reference program
# (oracle/_ref/gaussianMPI_ref: the reference sources compiled for sm_90a by `make -C oracle ref`,
# with the cutil.h / single-rank mpi.h shims) on an H100, from the repository root:
#   bash tests/golden/make_ref_golden.sh OUT_DIR
# then copy OUT_DIR/ref_c1* into tests/golden/ and commit.
set -euo pipefail
OUT=${1:?output directory}
mkdir -p "$OUT"
python - "$OUT" <<'PY'
import sys, os
sys.path.insert(0, os.getcwd())
import __graft_entry__ as e
pkg = e.load_package()
cfg = pkg.synth.CONFIGS["c1"]
ev = pkg.synth.make_blobs(cfg["N"], cfg["D"], cfg["K"])
pkg.synth.write_bin(os.path.join(sys.argv[1], "c1.bin"), ev)
PY
export OMP_NUM_THREADS=1 CUDA_VISIBLE_DEVICES=0
# config 1 with the shipped 100 iterations: checked by tests/test_oracle.py (first 512 events)
GMM_REF_ITERS=100 ./oracle/_ref/gaussianMPI_ref 8 "$OUT/c1.bin" "$OUT/ref_c1" 8 > "$OUT/ref_c1.stdout" 2>&1
head -n 512 "$OUT/ref_c1.results" > "$OUT/ref_c1.results.head"
rm -f "$OUT/ref_c1.results"
printf "N=10000\nD=4\nK=8\nseed=20260921\niters=100\n" > "$OUT/ref_c1.meta"
# 20 iterations: checked by tests/test_gpu_parity.py against the oracle and the engine (responsibilities of the first 2000 events)
GMM_REF_ITERS=20 ./oracle/_ref/gaussianMPI_ref 8 "$OUT/c1.bin" "$OUT/ref_c1_it20" 8 > /dev/null 2>&1
python - "$OUT" <<'PY'
import sys, os
import numpy as np
out = sys.argv[1]
rows = [l.rstrip("\n").split("\t") for l in open(os.path.join(out, "ref_c1_it20.results"))][:2000]
np.save(os.path.join(out, "ref_c1_it20.memberships.npy"), np.array([[float(v) for v in r[1].split(",")] for r in rows]))
PY
rm -f "$OUT/ref_c1_it20.results" "$OUT/c1.bin"
ls -la "$OUT"
