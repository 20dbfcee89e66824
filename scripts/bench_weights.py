"""EM throughput with and without per-event weights (gmm_set_weights) at c3: N = 10M, D = 24, K = 64 (synth.make_blobs).

Three runs on one context, alternated --repeats times: no weights; weights of one positive value (0.5, every fifth event
0), which the weighted wgmma M-step serves; and fractional weights uniform in [0.5, 1], which the FP64 SIMT M-step
serves (the tensor M-step admits one positive value only, DESIGN §5.11).  Each run is gmm_set_weights, gmm_seed,
gmm_estep, one warm-up gmm_em_iterations(K, 3), then gmm_em_iterations(K, --iters) timed with the host clock (the call
ends in a stream synchronisation); EM it/s is the best of the repeats, with the E- and M-step ms per iteration from
gmm_get_profile.  Prints the card's name, power limit and maximum SM clock (read-only nvidia-smi query) first.

    python scripts/bench_weights.py [--n 10000000] [--D 24] [--K 64] [--iters 20] [--repeats 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--D", type=int, default=24)
    ap.add_argument("--K", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    print(f"card: {card()}", flush=True)
    pkg = entry.load_package()
    pkg.load_library()
    ev = pkg.synth.make_blobs(a.n, a.D, a.K)
    rng = np.random.default_rng(1)
    one = np.full(a.n, 0.5, np.float32)
    one[::5] = 0.0
    runs = {"unweighted": None, "one_value": one, "fractional": rng.uniform(0.5, 1.0, a.n).astype(np.float32)}
    best = {k: None for k in runs}
    with pkg.Engine(ev, a.K) as eng:
        for _ in range(a.repeats):
            for name, w in runs.items():
                eng.set_weights(w)
                eng.seed(a.K)
                eng.estep(a.K)
                eng.em_iterations(a.K, 3)
                eng.profile(reset=True)
                t0 = time.perf_counter()
                eng.em_iterations(a.K, a.iters)
                dt = time.perf_counter() - t0
                p = eng.profile(reset=True)
                r = dict(it_s=a.iters / dt, estep_ms=p["estep_ms"] / a.iters, mstep_ms=p["mstep_ms"] / a.iters,
                         mstep="tensor" if p["mstep_tensor_launches"] else "simt")
                if best[name] is None or r["it_s"] > best[name]["it_s"]:
                    best[name] = r
    for name, r in best.items():
        print(json.dumps(dict(run=name, n=a.n, D=a.D, K=a.K, **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()})))
    print(f"one-value weights / unweighted: {best['one_value']['it_s'] / best['unweighted']['it_s']:.4f}")


if __name__ == "__main__":
    main()
