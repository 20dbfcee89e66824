"""Cost of gmm_condition: fit on 10M synth.make_blobs events, then score 10M fresh events measured on the first n_obs
dimensions and impute the others (mean and variance), at (D, K, n_obs) = (24, 64, 16), (16, 32, 8) and (32, 512, 16).

Per shape: the kernel's time per 10M events (gmm_get_condition_profile, CUDA events around each chunk's kernel) beside the
FP32 floor computed from its FMAs (per event and cluster n_obs (n_obs + 1) / 2 + n_obs for the marginal logit, NM n_obs for
G dx and 4 NM for the running moments, at the data-sheet 33.5 T FMA/s of the H100 SXM; computed, not measured); the
host-to-host rate (host clock around gmm_condition, best of --repeats after one warm-up call); and the host time a float64
numpy restatement (tests/_condition_ref.py) takes on --numpy-n events, scaled to 10M.  Prints the card's name, power limit
and maximum SM clock (read-only nvidia-smi query) first.

With --mode stats it measures gmm_condition_stats on the same rows instead: the kernel time (prep + marginal E-step + M-step)
per 10M events (gmm_get_condition_stats_profile) beside the resident E- and M-step times per 10M events of the same context
(gmm_get_profile over --em EM iterations on the 10M fitted events), the M-step kernel that served the chunks, and the
host-to-host rate with and without memberships (host clock around the call, best of --repeats after one warm-up call).

    python scripts/bench_condition.py [--mode condition|stats] [--n 10000000] [--repeats 3] [--em 10] [--numpy-n 200000]
                                      [--shapes 24x64x16,16x32x8,32x512x16]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as entry  # noqa: E402
import _condition_ref as cref  # noqa: E402
from bench_seed import card  # noqa: E402

FMA_PER_S = 33.5e12                 # H100 SXM data sheet: 67 TFLOPS FP32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--em", type=int, default=10)
    ap.add_argument("--numpy-n", type=int, default=200_000)
    ap.add_argument("--shapes", default="24x64x16,16x32x8,32x512x16")
    ap.add_argument("--mode", choices=("condition", "stats"), default="condition")
    a = ap.parse_args()
    pkg = entry.load_package()
    pkg.load_library()
    print(f"card: {card()}", flush=True)
    for shape in a.shapes.split(","):
        D, K, n_obs = (int(v) for v in shape.split("x"))
        nm = D - n_obs
        obs = np.arange(n_obs, dtype=np.int32)
        fit = pkg.synth.make_blobs(a.n, D, K, seed=20260921)
        new = np.ascontiguousarray(pkg.synth.make_blobs(a.n, D, K, seed=20261015)[:, :n_obs])
        res = dict(n=a.n, D=D, K=K, n_obs=n_obs)
        if a.mode == "stats":
            print(json.dumps(stats_shape(pkg, a, fit, new, D, K, obs)), flush=True)
            continue
        with pkg.Engine(fit, K) as eng:
            eng.seed(K)
            eng.em(K, a.em, a.em)
            cl = eng.get_clusters(K)
            lab = np.empty(a.n, np.int32)
            mr = np.empty(a.n, np.float32)
            lp = np.empty(a.n, np.float32)
            mean = np.empty((a.n, nm), np.float32)
            var = np.empty((a.n, nm), np.float32)
            ptrs = [v.ctypes.data for v in (lab, mr, lp, mean, var)]
            call = lambda: eng.lib.gmm_condition(eng.h, K, obs.ctypes.data, n_obs, new.ctypes.data, a.n, *ptrs, None)  # noqa: E731
            assert call() == 0, eng.lib.gmm_last_error()                          # warm-up: buffers
            walls = []
            eng.condition_profile(reset=True)
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                rc = call()
                walls.append(time.perf_counter() - t0)
                assert rc == 0, eng.lib.gmm_last_error()
            prof = eng.condition_profile()
        kernel_ms = prof["kernel_ms"] / a.repeats * 1e7 / a.n
        fmas = K * (n_obs * (n_obs + 1) // 2 + n_obs + nm * n_obs + 4 * nm)
        floor_ms = fmas * 1e7 / FMA_PER_S * 1e3
        res.update(kernel_ms_per_10M=round(kernel_ms, 3), fp32_floor_ms_per_10M=round(floor_ms, 3),
                   floor_fraction=round(floor_ms / kernel_ms, 3), host_to_host_ms=round(min(walls) * 1e3, 1),
                   host_to_host_events_per_s=float(f"{a.n / min(walls):.3g}"),
                   kernel_share_of_host_to_host=round(prof["kernel_ms"] / a.repeats / (min(walls) * 1e3), 3))
        m = min(a.numpy_n, a.n)
        t0 = time.perf_counter()
        for s in range(0, m, 20_000):
            cref.condition(cl, K, obs, new[s:min(m, s + 20_000)])
        res["numpy_f64_ms_per_10M"] = round((time.perf_counter() - t0) * 1e3 * 1e7 / m, 0)
        print(json.dumps(res), flush=True)


def stats_shape(pkg, a, fit, new, D, K, obs):
    n_obs = len(obs)
    res = dict(mode="stats", n=a.n, D=D, K=K, n_obs=n_obs)
    with pkg.Engine(fit, K) as eng:
        eng.seed(K)
        eng.em(K, 2, 2)
        eng.profile(reset=True)
        eng.em_iterations(K, a.em)                  # the resident steps on the same context, for comparison
        p = eng.profile()
        res.update(resident_estep_ms_per_10M=round(p["estep_ms"] / a.em * 1e7 / a.n, 3),
                   resident_mstep_ms_per_10M=round(p["mstep_ms"] / a.em * 1e7 / a.n, 3))
        st = np.empty(pkg.stats_len(K, D), np.float64)
        sh = np.empty(D, np.float64)
        mb = np.empty((K, a.n), np.float32)
        for memberships in (False, True):
            call = lambda: eng.lib.gmm_condition_stats(eng.h, K, obs.ctypes.data, n_obs, new.ctypes.data, a.n, st.ctypes.data,  # noqa: E731
                                                       sh.ctypes.data, mb.ctypes.data if memberships else None)
            assert call() == 0, eng.lib.gmm_last_error()                          # warm-up: buffers
            eng.condition_stats_profile(reset=True)
            walls = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                rc = call()
                walls.append(time.perf_counter() - t0)
                assert rc == 0, eng.lib.gmm_last_error()
            prof = eng.condition_stats_profile()
            tag = "with_memberships" if memberships else "stats_only"
            if not memberships:
                res.update(kernel_ms_per_10M=round(prof["kernel_ms"] / a.repeats * 1e7 / a.n, 3),
                           mstep_tensor_chunks=prof["mstep_tensor_chunks"] // a.repeats,
                           mstep_simt_chunks=prof["mstep_simt_chunks"] // a.repeats)
            res[f"host_to_host_ms_{tag}"] = round(min(walls) * 1e3, 1)
            res[f"host_to_host_events_per_s_{tag}"] = float(f"{a.n / min(walls):.3g}")
    return res


if __name__ == "__main__":
    main()
