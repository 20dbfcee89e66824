"""Modal clustering (gmm_mode_labels, gmm_modes) on the GPU.

gmm_mode_labels over the c3 shard (N = 10M, D = 24, K = 64, synth.make_blobs) after gmm_seed and 20 EM iterations: wall and
kernel ms (gmm_get_modes_profile), mean and maximum iterations per event and their histogram, event-iterations per second and FLOP/s against
NVIDIA's 67 TFLOP/s FP32 data-sheet figure for the H100 SXM.  The FLOP model counts what mode_iter_kernel executes per
event-iteration at the padded dimension DP: per component DP (dx) + 2 DP^2 (v = S dx) + 2 DP (q) + 2 DP (g) + DP (DP + 1)
(A's packed lower triangle), then DP^3 / 3 + 2 DP^2 for the Cholesky factorisation and the two solves.  Then gmm_modes at
K = 512, D = 16 (1M events, 5 EM iterations).  Prints the card's name, power limit and maximum SM clock (read-only
nvidia-smi query) first.

    python scripts/bench_modes.py [--n 10000000] [--repeats 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import __graft_entry__ as entry  # noqa: E402
from bench_weights import card  # noqa: E402

FP32_PEAK = 67e12


def flops_per_event_iteration(D, K):
    DP = (D + 3) & ~3
    return K * (DP + 2 * DP * DP + 4 * DP + DP * (DP + 1)) + DP ** 3 / 3 + 2 * DP * DP


def labels(pkg, a):
    n, D, K = a.n, 24, 64
    ev = pkg.synth.make_blobs(n, D, K)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.estep(K)
        eng.em_iterations(K, 20)
        md = eng.modes(K)
        eng.mode_labels(K, md["modes"], max_iter=a.max_iter)            # warm-up
        best = None
        for _ in range(a.repeats):
            eng.modes_profile(reset=True)
            t0 = time.perf_counter()
            got = eng.mode_labels(K, md["modes"], max_iter=a.max_iter, iters=True)
            wall = (time.perf_counter() - t0) * 1e3
            pr = eng.modes_profile(reset=True)
            if best is None or wall < best[0]:
                best = (wall, pr, got)
        wall, pr, got = best
        ei = int(got["iters"].sum())
        fl = ei * flops_per_event_iteration(D, K)
        print(json.dumps(dict(call="gmm_mode_labels", n=n, D=D, K=K, n_modes=len(md["modes"]), wall_ms=round(wall, 2),
                              kernel_ms=round(pr["kernel_ms"], 2), mean_iters=round(float(got["iters"].mean()), 2),
                              max_iters=int(got["iters"].max()),
                              iters_histogram={int(i): int(c) for i, c in enumerate(np.bincount(got["iters"])) if c},
                              unmatched=got["unmatched"], unconverged=got["unconverged"],
                              event_iterations_per_s=ei / (pr["kernel_ms"] / 1e3), tflops=fl / (pr["kernel_ms"] / 1e3) / 1e12,
                              fp32_peak_frac=fl / (pr["kernel_ms"] / 1e3) / FP32_PEAK)), flush=True)


def modes(pkg, a):
    n, D, K = 1_000_000, 16, 512
    ev = pkg.synth.make_blobs(n, D, 64)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.estep(K)
        eng.em_iterations(K, 5)
        eng.modes(K)
        best = None
        for _ in range(a.repeats):
            eng.modes_profile(reset=True)
            t0 = time.perf_counter()
            md = eng.modes(K)
            wall = (time.perf_counter() - t0) * 1e3
            pr = eng.modes_profile(reset=True)
            if best is None or wall < best[0]:
                best = (wall, pr, md)
        wall, pr, md = best
        print(json.dumps(dict(call="gmm_modes", D=D, K=K, n_modes=len(md["modes"]), wall_ms=round(wall, 2),
                              kernel_ms=round(pr["kernel_ms"], 2), max_iters=int(md["iters"].max()),
                              maxima=int(md["is_max"].sum()))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--max-iter", type=int, default=500)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    pkg = entry.load_package()
    pkg.load_library()
    print(json.dumps(card()), flush=True)
    modes(pkg, a)
    labels(pkg, a)


if __name__ == "__main__":
    main()
