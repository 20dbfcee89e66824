"""Cost and benefit of gmm_seed_kmeans against gmm_seed at N = 10M, D = 24, K = 64 (synth.make_blobs, 64 blobs).

Times (host clock around calls that end in a stream synchronisation, best of --repeats after one warm-up call):
gmm_seed, gmm_seed_kmeans with max_iter 0 (k-means++, one assignment, one M-step) and with max_iter 20, so that the
differences separate k-means++ from Lloyd.  Then the log-likelihood after gmm_em(K, 100, 100) from each seeding, on the
shuffled data and on the same data sorted by blob (the nearest generating centre).  Prints the card's name, power limit
and maximum SM clock (read-only nvidia-smi query) first.

    python scripts/bench_seed.py [--n 10000000] [--D 24] [--K 64] [--repeats 3] [--em 100]
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


def best_ms(fn, repeats):
    fn()                                         # warm-up: buffers, kernel attributes
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--D", type=int, default=24)
    ap.add_argument("--K", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--em", type=int, default=100)
    a = ap.parse_args()
    pkg = entry.load_package()
    pkg.load_library()
    print(f"card: {card()}", flush=True)
    seed = 20260921
    x = pkg.synth.make_blobs(a.n, a.D, a.K, seed=seed)
    res = dict(n=a.n, D=a.D, K=a.K)
    with pkg.Engine(x, a.K) as eng:
        res["seed_ms"] = best_ms(lambda: eng.seed(a.K), a.repeats)
        it = {}
        for m in (0, 20):
            res[f"kmeans_it{m}_ms"] = best_ms(lambda: it.__setitem__(m, eng.seed_kmeans(a.K, max_iter=m, seed=0)[2]), a.repeats)
            res[f"kmeans_it{m}_updates"] = it[m]
        res["lloyd_ms_per_update"] = (res["kmeans_it20_ms"] - res["kmeans_it0_ms"]) / max(1, it[20])
    print(json.dumps(res), flush=True)
    centres = np.random.default_rng(seed).uniform(-10.0, 10.0, size=(a.K, a.D))   # make_blobs' first draws
    own = np.empty(a.n, np.int64)
    for s in range(0, a.n, 1 << 20):
        xs = x[s:s + (1 << 20)].astype(np.float64)
        own[s:s + len(xs)] = np.argmin((xs * xs).sum(1)[:, None] - 2 * xs @ centres.T + (centres * centres).sum(1)[None], 1)
    for order in ("shuffled", "sorted"):
        xo = x if order == "shuffled" else np.ascontiguousarray(x[np.argsort(own, kind="stable")])
        out = dict(order=order)
        with pkg.Engine(xo, a.K) as eng:
            for name, seeding in (("seed", lambda: eng.seed(a.K)),
                                  ("kmeans_it0", lambda: eng.seed_kmeans(a.K, max_iter=0, seed=0)),
                                  ("kmeans_it20", lambda: eng.seed_kmeans(a.K, max_iter=20, seed=0))):
                seeding()
                ll, iters = eng.em(a.K, a.em, a.em)
                means = eng.get_clusters(a.K).means[:a.K].astype(np.float64)
                owner = np.argmin(((means[:, None, :] - centres[None]) ** 2).sum(-1), 1)
                out[f"{name}_loglik"] = ll
                out[f"{name}_blobs_missed"] = a.K - len(set(owner.tolist()))
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
