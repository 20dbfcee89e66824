"""EM over several samples (gmm_em_multisample) against pooled EM (gmm_em_iterations).

At c3's shape (N = 10M, D = 24, K = 64, synth.make_blobs) cut into S in {1, 16, 256} equal samples, and at K = 512 with
1M events: multi-sample iterations per second (min = max = --iters, from gmm_seed) against gmm_em_iterations from the same
start, best of --repeats; per iteration the reweight pass's kernel ms (reweight + finishing kernel, gmm_get_multisample_profile)
against its HBM bound (read and write 4 K bytes per event at 3.35 TB/s) and the host ms of the finalisation and the pi / rho
update.  Prints the card's name, power limit and maximum SM clock (read-only nvidia-smi query) first.

    python scripts/bench_multisample.py [--n 10000000] [--iters 20] [--repeats 3]
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


def run(pkg, n, D, K, samples, a):
    ev = pkg.synth.make_blobs(n, D, min(K, 64))
    with pkg.Engine(ev, K) as eng:
        for S in samples:
            off = np.linspace(0, n, S + 1).astype(np.int64)
            pi0 = np.full((S, K), 1.0 / K)                   # equal rows: every pass is a full reweight
            best = {}
            for _ in range(a.repeats):
                eng.seed(K)
                eng.estep(K)
                eng.em_iterations(K, 3)
                t0 = time.perf_counter()
                eng.em_iterations(K, a.iters)
                em = a.iters / (time.perf_counter() - t0)
                eng.seed(K)
                eng.em_multisample(K, off, pi0, 3, 3)
                eng.seed(K)
                eng.multisample_profile(reset=True)
                t0 = time.perf_counter()
                _, _, _, it, _ = eng.em_multisample(K, off, pi0, a.iters, a.iters)
                dt = time.perf_counter() - t0
                pr = eng.multisample_profile(reset=True)
                # a call runs iters + 1 E-steps and reweight passes and iters M-steps
                r = dict(em_it_s=em, ms_it_s=it / dt, pass_ms=pr["kernel_ms"] / (it + 1), host_ms=pr["host_ms"] / it,
                         pass_hbm_bound_ms=8.0 * K * n / 3.35e12 * 1e3)
                if not best or r["ms_it_s"] > best["ms_it_s"]:
                    best = r
            print(json.dumps(dict(n=n, D=D, K=K, S=S, **{k: round(v, 3) for k, v in best.items()})), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    pkg = entry.load_package()
    pkg.load_library()
    print(json.dumps(card()), flush=True)
    run(pkg, a.n, 24, 64, (1, 16, 256), a)
    run(pkg, 1_000_000, 24, 512, (16,), a)


if __name__ == "__main__":
    main()
