"""Throughput of gmm_score: fit parameters on 10M training events (seed + EM iterations), then score 10M fresh events
from the same seeded generator, at (D, K) = (24, 64), (24, 128) and (16, 32).

Reported per shape: the score kernel's time per 10M events and its events/s (device only; bound by the tensor or FP32
pipe like the E-step, which reads the same 4 D bytes per event but writes 4 K bytes instead of 12), the host-to-host
rate through gmm_score (4 D bytes in and 12 bytes out per event over PCIe, plus the host copies into and out of the
pinned stages: expected to be bound by those copies), and the E-step's time at the same shape from gmm_get_profile.
Prints the card's name, power limit and maximum SM clock (read-only nvidia-smi query) first.

--mode stats times gmm_score_stats instead, once with statistics only and once with memberships as well: the kernel time
(prep + E-step + M-step) per 10M events, the host-to-host rate (4 D bytes in per event, plus 4 K bytes out with
memberships), the per-chunk wait of the compute stream for the range flag, and the resident E-step + M-step time at the
same shape from gmm_get_profile.

    python scripts/bench_score.py [--mode score|stats] [--n 10000000] [--iters 5] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as entry  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:                       # noqa: BLE001
        return f"unknown ({e})"


def bench_shape(pkg, train, fresh, K, iters, repeats):
    n, D = fresh.shape
    with pkg.Engine(train, K) as eng:
        eng.seed(K)
        eng.estep(K)
        eng.em_iterations(K, iters)
        eng.profile(reset=True)
        for _ in range(repeats):
            eng.estep(K)
        estep_ms = eng.profile()["estep_ms"] / repeats
        eng.score(K, fresh[: min(n, 1 << 20)], max_resp=False)        # warm-up: buffers, kernel attributes
        kern, h2h = [], []
        for _ in range(repeats):
            eng.score_profile(reset=True)
            t0 = time.perf_counter()
            eng.score(K, fresh)
            wall = time.perf_counter() - t0
            p = eng.score_profile()
            kern.append(p["kernel_ms"])
            h2h.append(wall)
            path = "wgmma" if p["tensor_chunks"] and not p["simt_chunks"] else ("SIMT" if not p["tensor_chunks"] else "mixed")
    k_ms = float(np.median(kern)) * 1e7 / n
    wall_s = float(np.median(h2h))
    return dict(D=D, K=K, path=path, score_kernel_ms_per_10M=round(k_ms, 3), score_kernel_events_per_s=round(1e7 / (k_ms * 1e-3)),
                host_to_host_events_per_s=round(n / wall_s), host_to_host_ms=round(wall_s * 1e3, 1),
                estep_ms_per_10M=round(estep_ms * 1e7 / train.shape[0], 3))


def bench_stats_shape(pkg, train, fresh, K, iters, repeats):
    n, D = fresh.shape
    with pkg.Engine(train, K) as eng:
        eng.seed(K)
        eng.estep(K)
        eng.em_iterations(K, iters)
        eng.profile(reset=True)
        for _ in range(repeats):
            eng.estep(K)
            eng.mstep(K)
            eng.constants(K)
        prof = eng.profile()
        estep_ms, mstep_ms = prof["estep_ms"] / repeats, prof["mstep_ms"] / repeats
        eng.score_stats(K, fresh[: min(n, 1 << 20)], memberships=True)     # warm-up: buffers, pinned mirror, attributes
        out = dict(D=D, K=K, resident_estep_ms_per_10M=round(estep_ms * 1e7 / train.shape[0], 3),
                   resident_mstep_ms_per_10M=round(mstep_ms * 1e7 / train.shape[0], 3))
        for memb in (False, True):
            kern, wall, wait, nchunks = [], [], [], 0
            for _ in range(repeats):
                eng.score_stats_profile(reset=True)
                t0 = time.perf_counter()
                eng.score_stats(K, fresh, memberships=memb)
                wall.append(time.perf_counter() - t0)
                p = eng.score_stats_profile()
                kern.append(p["kernel_ms"])
                wait.append(p["flag_wait_ms"])
                nchunks = p["estep_tensor_chunks"] + p["estep_simt_chunks"]
                path = f"E {'wgmma' if not p['estep_simt_chunks'] else 'SIMT/mixed'}, M {'wgmma' if not p['mstep_simt_chunks'] else 'FP64/mixed'}"
            tag = "memb" if memb else "stats"
            out[f"{tag}_path"] = path
            out[f"{tag}_kernel_ms_per_10M"] = round(float(np.median(kern)) * 1e7 / n, 3)
            out[f"{tag}_host_to_host_events_per_s"] = round(n / float(np.median(wall)))
            out[f"{tag}_flag_wait_ms_per_chunk"] = round(float(np.median(wait)) / max(nchunks, 1), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--mode", default="score", choices=["score", "stats"])
    a = ap.parse_args()
    pkg = entry.load_package()
    pkg.load_library()
    print("card:", card(), flush=True)
    data = {}
    for D, K in ((24, 64), (24, 128), (16, 32)):
        if D not in data:                        # training and fresh events: disjoint halves of one seeded draw
            both = pkg.synth.make_blobs(2 * a.n, D, 16, seed=1)
            data = {D: (np.ascontiguousarray(both[:a.n]), np.ascontiguousarray(both[a.n:]))}
            del both
        train, fresh = data[D]
        bench = bench_shape if a.mode == "score" else bench_stats_shape
        print(json.dumps(bench(pkg, train, fresh, K, a.iters, a.repeats)), flush=True)


if __name__ == "__main__":
    main()
