"""Cost of gmm_sample: fit on 10M synth.make_blobs events, then draw 10M events from the fit, at (D, K) = (24, 64),
(16, 32) and (32, 512).

Per shape: the sampling kernel's time per 10M events (gmm_get_sample_profile, CUDA events around each chunk's kernel)
with its fraction of the HBM bound (4 (D + 1) bytes written per event at 3.35 TB/s); the host-to-host rate (host clock
around gmm_sample, best of --repeats after one warm-up call); and, for comparison, the host time numpy takes to draw the
same number of events from the same mixture (sklearn's way: multinomial counts, then per component z L^T + mu).  Prints
the card's name, power limit and maximum SM clock (read-only nvidia-smi query) first.

    python scripts/bench_sample.py [--n 10000000] [--repeats 3] [--em 10] [--shapes 24x64,16x32,32x512]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as entry  # noqa: E402
from bench_seed import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def numpy_sample(cl, K, n, rng):
    pi = cl.pi[:K].astype(np.float64)
    counts = rng.multinomial(n, pi / pi.sum())
    out = np.empty((n, cl.D), np.float32)
    pos = 0
    for k in range(K):
        L = np.linalg.cholesky(cl.R[k].astype(np.float64))
        m = int(counts[k])
        out[pos:pos + m] = rng.standard_normal((m, cl.D)) @ L.T + cl.means[k]
        pos += m
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--em", type=int, default=10)
    ap.add_argument("--shapes", default="24x64,16x32,32x512")
    a = ap.parse_args()
    pkg = entry.load_package()
    pkg.load_library()
    print(f"card: {card()}", flush=True)
    for shape in a.shapes.split(","):
        D, K = (int(v) for v in shape.split("x"))
        x = pkg.synth.make_blobs(a.n, D, K, seed=20260921)
        res = dict(n=a.n, D=D, K=K)
        with pkg.Engine(x, K) as eng:
            eng.seed(K)
            eng.em(K, a.em, a.em)
            cl = eng.get_clusters(K)
            out = np.empty((a.n, D), np.float32)
            lab = np.empty(a.n, np.int32)
            eng.lib.gmm_sample(eng.h, K, a.n, 1, 0, out.ctypes.data, lab.ctypes.data)   # warm-up: buffers, attributes
            walls = []
            eng.sample_profile(reset=True)
            for r in range(a.repeats):
                t0 = time.perf_counter()
                rc = eng.lib.gmm_sample(eng.h, K, a.n, 2 + r, 0, out.ctypes.data, lab.ctypes.data)
                walls.append(time.perf_counter() - t0)
                assert rc == 0, pkg.load_library().gmm_last_error()
            prof = eng.sample_profile()
        kernel_ms = prof["kernel_ms"] / a.repeats * 1e7 / a.n
        bound_ms = 4.0 * (D + 1) * 1e7 / HBM_BYTES_PER_S * 1e3
        res.update(kernel_ms_per_10M=round(kernel_ms, 3), hbm_bound_ms_per_10M=round(bound_ms, 3),
                   kernel_fraction_of_bound=round(bound_ms / kernel_ms, 3),
                   host_to_host_ms=round(min(walls) * 1e3, 1), host_to_host_events_per_s=float(f"{a.n / min(walls):.3g}"),
                   kernel_share_of_host_to_host=round(prof["kernel_ms"] / a.repeats / (min(walls) * 1e3), 3))
        rng = np.random.default_rng(0)
        t0 = time.perf_counter()
        numpy_sample(cl, K, a.n, rng)
        res["numpy_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
