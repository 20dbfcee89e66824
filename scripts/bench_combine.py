"""Cost of combining mixture components (gmm_combine, gmm_combine_labels).

At c3 (N = 10M, D = 24, K = 64, synth.make_blobs) after 20 EM iterations from gmm_seed: gmm_combine's wall and kernel ms
(best of --repeats, gmm_get_combine_profile), then one call under torch.profiler for each pass's device time: the all-pairs
pass against its K(K-1)/2 n pair evaluations and its one-read byte bound (4 K n bytes at 3.35 TB/s), the K-2 step passes
against their sum_L (L-1) n pair evaluations and K-2 reads of all K rows (4 K n bytes each), and gmm_combine_labels at
16 clusters against its 4 K n byte bound.  Then K = 128 and K = 512 at --n-small events (D = 16, after gmm_seed and one
E-step).  Prints the card's name, power limit and maximum SM clock (read-only nvidia-smi query) first.

    python scripts/bench_combine.py [--n 10000000] [--n-small 1000000] [--repeats 3]
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

HBM = 3.35e12


def device_ms_by_kernel(fn):
    """Device time per kernel name (ms) of one fn() call, from torch.profiler's CUDA activities."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        for key in ("combine_pairs_kernel", "combine_step_kernel", "combine_labels_kernel", "combine_sum_ranges_kernel",
                    "resp_entropy_kernel"):
            if key in ev.name:
                out[key] = out.get(key, 0.0) + ev.device_time_total / 1e3
    return out


def run(pkg, n, D, K, em_iters, repeats, seed):
    ev = pkg.synth.make_blobs(n, D, min(K, 64), seed=seed)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.estep(K)
        if em_iters:
            eng.em_iterations(K, em_iters)
        eng.combine(K)                                            # warm-up: buffers, modules
        best = None
        for _ in range(repeats):
            eng.combine_profile(reset=True)
            t0 = time.perf_counter()
            r = eng.combine(K)
            wall = (time.perf_counter() - t0) * 1e3
            p = eng.combine_profile(reset=True)
            if best is None or wall < best[0]:
                best = (wall, p["kernel_ms"])
        grp = pkg.host_combine_groups(r["merges"], K, min(16, K))
        eng.combine_labels(K, grp)
        lab_wall = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            eng.combine_labels(K, grp, max_sum=False)
            lab_wall.append((time.perf_counter() - t0) * 1e3)
        dev = device_ms_by_kernel(lambda: (eng.combine(K), eng.combine_labels(K, grp, max_sum=False)))
    pairs1 = K * (K - 1) // 2 * n
    pairs_steps = sum(L - 1 for L in range(2, K)) * n           # after merge s the merged group meets L - 1 = K - s - 2 others
    row_bytes = 4.0 * K * n
    out = dict(n=n, D=D, K=K, em_iters=em_iters, combine_wall_ms=best[0], combine_kernel_ms=best[1],
               pairs_ms=dev.get("combine_pairs_kernel", 0.0), pairs_evals=pairs1,
               pairs_gevals_s=pairs1 / max(dev.get("combine_pairs_kernel", 0.0), 1e-9) / 1e6, pairs_hbm_bound_ms=row_bytes / HBM * 1e3,
               steps=K - 2, steps_ms=dev.get("combine_step_kernel", 0.0), steps_evals=pairs_steps,
               steps_hbm_bound_ms=(K - 2) * row_bytes / HBM * 1e3,
               steps_gb_s=(K - 2) * row_bytes / max(dev.get("combine_step_kernel", 0.0), 1e-9) / 1e6,
               sums_ms=dev.get("combine_sum_ranges_kernel", 0.0), entropy_ms=dev.get("resp_entropy_kernel", 0.0),
               labels_ms=dev.get("combine_labels_kernel", 0.0), labels_hbm_bound_ms=row_bytes / HBM * 1e3,
               labels_wall_ms=min(lab_wall))
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in out.items()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--n-small", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    print(f"card: {card()}", flush=True)
    pkg = entry.load_package()
    pkg.load_library()
    run(pkg, a.n, 24, 64, 20, a.repeats, 1)
    run(pkg, a.n_small, 16, 128, 0, a.repeats, 2)
    run(pkg, a.n_small, 16, 512, 0, max(1, a.repeats // 3), 3)


if __name__ == "__main__":
    main()
