"""Error model of the tensor M-step (`mstep_tc_kernel<D>`, csrc/kernels_tc.cu), on the CPU, numpy only.

The emulator below repeats the kernel's operand arithmetic bit for bit where it is exact and to within the FP32 accumulation
of the tensor cores where it is not:
  * z = fl32(fl32(x - shift) * inv_scale), the standardised copy the kernel reads;
  * quanta q = zb * 2^-11 for the coordinate rows and zb^2 * 2^-11 for the product rows (zb = power-of-two bound of |z| over
    all dimensions, tc_set_shift_scale), p_h = q * round(phi / q) from the exact value, p_l = fp16(fl32(phi - p_h));
  * g_h = 2^-6 * round(2^6 g), g_l = fp16(1024 (g - g_h)) / 1024, g_s = fp16(1024 g) / 1024;
  * per CTA (the event ranges of launch_mstep_d()) and feature tile (the operand row map of tc_row_info()), the exact group
    sum p_h g_h per 128-event chain and the remainder group sum p_h g_l + p_l g_s per 512-event chain, both staggered by the
    tile index, drained into one FP32 round-to-nearest partial sum per statistic and cluster; the CTAs' partials summed in
    double and un-scaled.
The remainder chains are summed exactly and rounded to FP32 once at the drain: the tensor cores' truncating accumulation of
those (~1 % of the statistic) is the only part not emulated.

The per-cluster bar (MSTEP_TOL below: 1.5e-5 on N, 1e-5 on the means and on R) compares N, the means and R of one
M-step with the exact-arithmetic M-step on the same responsibilities.  Means and R are measured against the cluster's raw
second moment about the centre, M2 = max_i (R_ii + (mu_i - s_i)^2), so that the bar does not depend on how far the cluster
sits from the centre.  The faithful scheme's worst errors over the shapes below are 2.9e-6 on N, 2.1e-6 on the means and
1.6e-6 on R, all from clusters made mostly of events with small g: the FP16 rounding of g_l (relative 2^-12) dominates
there.  The FP16 remainder p_l grows with the product quantum zb^2 * 2^-11: one event just under 64 standard deviations
(zb = 64) raises the error on R of 200 000 blob events from 2.5e-8 to 1.4e-6, still below a quarter of the bar, which is
therefore not widened for the worst legal range.

This module asserts that the faithful scheme stays at or below a quarter of the bar at the shapes the GPU tests
(tests/test_gpu_mstep_tc.py) run, and that each of these kernel faults exceeds the bar at one of them at least:
  * drop_pl_gs   — the p_l g_s product dropped: up to 350 times the bar;
  * pl_gh        — p_l g_h used in place of p_l g_s (an earlier build): at most 3.6e-5 on R, 1.1e-5 on the means;
  * drop_ph_gl   — the p_h g_l product dropped: up to 2e4 times the bar (N off by 1e-2 .. 2e-1);
  * no_last_rem  — the remainder group's last partial chain of each CTA never drained (a drain bug at i == nsub - 1):
                   at every shape with fewer than 512 events per CTA that is the whole remainder group, as bad as drop_ph_gl.
Run it as a script (python tests/test_mstep_error_model.py) for the table of errors per shape.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import entry  # noqa: E402

KTE, CHAIN, CHAIN2, PHI_BITS = 32, 4, 16, 11          # sub-tile events, sub-tiles per exact / remainder chain, |p_h| <= 2^11 q
H100_SMS = 132                                        # H100 SXM5: CTAs of the M-step grid row
VARIANTS = ("faithful", "drop_pl_gs", "pl_gh", "drop_ph_gl", "no_last_rem")


# Per-cluster bar of ONE tensor M-step against the exact-arithmetic M-step on the same responsibilities (derived and
# checked against kernel faults by the tests below).  N is relative; means and R are relative to the
# cluster's raw second moment about the centre s, M2 = max_i (R_ii + (mu_i - s_i)^2) (sqrt(M2) for the means).
MSTEP_TOL = dict(N=1.5e-5, mean=1e-5, R=1e-5)


def finalize_np(stats, shift, K, D):
    """N, means, R [K][D][D] from packed statistics about `shift` (float64, avgvar 0)."""
    s = np.asarray(stats, np.float64)[:K * (1 + D + D * (D + 1) // 2)].reshape(K, -1)
    N = s[:, 0]
    m = s[:, 1:1 + D] / np.where(N != 0, N, 1.0)[:, None]
    S2 = np.zeros((K, D, D))
    i, j = np.tril_indices(D)                  # row by row: the packed order i(i+1)/2 + j of host_math.h feat2
    S2[:, i, j] = s[:, 1 + D:]
    S2[:, j, i] = s[:, 1 + D:]
    R = (S2 - m[:, :, None] * s[:, None, 1:1 + D]) / np.where(N > 0, N, 1.0)[:, None, None]
    return N, m + shift, R


def param_errors(N, mu, R, N_ref, mu_ref, R_ref, shift):
    """Worst per-cluster deviations of (N, means, R) from the reference, in the units of MSTEP_TOL, and their worst
    ratio to the bar ("worst" <= 1: within the bar).  Clusters with N_ref < 1 (R zeroed) are not measured."""
    N, mu, R, N_ref, mu_ref, R_ref = (np.asarray(a, np.float64) for a in (N, mu, R, N_ref, mu_ref, R_ref))
    shift = np.asarray(shift, np.float64)
    eN = float((np.abs(N - N_ref) / np.maximum(N_ref, 1.0)).max())
    live = N_ref >= 1.0
    M2 = (np.diagonal(R_ref, axis1=1, axis2=2) + (mu_ref - shift) ** 2).max(1)[live]
    em = float((np.abs(mu - mu_ref)[live].max(1) / np.sqrt(M2)).max()) if live.any() else 0.0
    eR = float((np.abs(R - R_ref)[live].max((1, 2)) / M2).max()) if live.any() else 0.0
    worst = max(eN / MSTEP_TOL["N"], em / MSTEP_TOL["mean"], eR / MSTEP_TOL["R"])
    return dict(N=eN, mean=em, R=eR, worst=worst)


def mstep_errors(stats, stats_ref, shift, K):
    """param_errors() of two sets of packed statistics about the same shift."""
    D = len(shift)
    return param_errors(*finalize_np(stats, shift, K, D), *finalize_np(stats_ref, shift, K, D), shift)


def exact_mstep_stats(events, gamma, shift):
    """Packed statistics [K * F + 1] (S0 | S1 | S2 lower triangle per cluster, then the log-likelihood slot) of the
    float32 events weighted by the float32 responsibilities [K][N], about `shift`, in float64."""
    y = np.asarray(events, np.float32).astype(np.float64) - np.asarray(shift, np.float64)
    g = np.asarray(gamma, np.float32).astype(np.float64)
    D = y.shape[1]
    i, j = np.tril_indices(D)
    rows = []
    for k in range(len(g)):
        S2 = (g[k][:, None] * y).T @ y
        rows.append(np.concatenate([[g[k].sum()], g[k] @ y, S2[i, j]]))
    return np.concatenate(rows + [[0.0]])


def f16(a):
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


def f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def pairs(D):
    """(i, j), i >= j, in the packed order of the second-moment statistics (host_math.h feat2)."""
    return np.array([(i, j) for i in range(D) for j in range(i + 1)], np.int64).reshape(-1, 2)


def feature_tiles(D):
    """Feature tile (128 operand rows each) that produces each packed statistic: the row map of tc_row_info()."""
    S, half = D // 4, D // 2
    RPP = 1 + 2 * S + S * half
    CPP = (RPP + 7) // 8
    F = 1 + D + D * (D + 1) // 2
    tile = np.full(F, -1)
    for row in range(4 * CPP * 8):
        p, r = divmod(row, CPP * 8)
        if r >= RPP:
            continue
        if r == 0:
            f = 0 if p == 0 else -1
        elif r <= S:
            f = 1 + (r - 1 + p * S) % D
        else:
            if r <= 2 * S:
                a = b = r - 1 - S
            else:
                t = r - 1 - 2 * S
                a, b = t // half, (t // half + 1 + t % half) % D
            ta, tb = (a + p * S) % D, (b + p * S) % D
            if a != b and (b - a) % D == half and ta >= half:
                f = -1
            else:
                i, j = max(ta, tb), min(ta, tb)
                f = 1 + D + i * (i + 1) // 2 + j
        if f >= 0:
            assert tile[f] < 0, "row map: a statistic is produced twice"
            tile[f] = row // 128
    assert (tile >= 0).all(), "row map: a statistic is not produced"
    return tile


def cta_ranges(n, n_sms):
    """launch_mstep_d(): events per CTA (a multiple of the 32-event sub-tile) and the number of CTAs per grid row."""
    per = -(-n // n_sms)
    per = -(-per // KTE) * KTE
    return per, -(-n // per)


def standardise(x):
    """shift, inv_scale and z exactly as ensure_moments() + tc_set_shift_scale() form them, and the bound zb."""
    xd = x.astype(np.float64)
    mean = xd.sum(0) / len(xd)
    var = (xd * xd).sum(0) / len(xd) - mean * mean
    scale = np.where(var > 0, np.sqrt(np.maximum(var, 0)), 1.0)
    sf = mean.astype(np.float32)
    isf = (1.0 / scale).astype(np.float32)
    z = ((x.astype(np.float32) - sf) * isf).astype(np.float32)
    za = np.maximum(np.abs(xd.max(0) - sf), np.abs(xd.min(0) - sf)) * isf.astype(np.float64) * (1 + 1e-6)
    zmax = np.where(za > 0, np.ldexp(1.0, np.frexp(za)[1]), 1.0)
    return sf.astype(np.float64), 1.0 / isf.astype(np.float64), z.astype(np.float64), float(zmax.max())


def emulate(x, g, n_sms=H100_SMS, variants=VARIANTS):
    """Packed statistics [K][F] about the kernel's shift, as each variant of the kernel would produce them."""
    N, D = x.shape
    K = g.shape[0]
    shift, scale, z, zb = standardise(x)
    ql, qp = zb / 2 ** PHI_BITS, zb * zb / 2 ** PHI_BITS
    P = pairs(D)
    F = 1 + D + len(P)
    tile = feature_tiles(D)
    per, gx = cta_ranges(N, n_sms)
    nsub = np.array([-(-(min(N, (c + 1) * per) - c * per) // KTE) for c in range(gx)])
    ex = np.zeros((gx, F, K))
    rm = {v: np.zeros((gx, F, K)) for v in variants}
    racc = {v: np.zeros((gx, F, K), np.float32) for v in variants}
    g64 = g.astype(np.float64)
    for s in range(int(nsub.max())):
        idx = np.arange(gx)[:, None] * per + s * KTE + np.arange(KTE)[None, :]
        ok = idx < np.minimum(N, (np.arange(gx)[:, None] + 1) * per)
        idx = np.where(ok, idx, 0)
        zc = np.where(ok[..., None], z[idx], 0.0)
        gc = np.where(ok[None], g64[:, idx], 0.0).transpose(1, 2, 0)          # [cta][event][cluster]
        lin = zc
        prod = zc[..., P[:, 0]] * zc[..., P[:, 1]]
        hl = np.round(lin / ql) * ql
        hp = np.round(prod / qp) * qp
        ph = np.concatenate([np.ones(zc.shape[:2] + (1,)), hl, hp], axis=2)
        pl = np.concatenate([np.zeros(zc.shape[:2] + (1,)), f16(f32(lin - hl)), f16(f32(prod - hp))], axis=2)
        gh = np.round(gc * 64.0) / 64.0
        gl = f16(1024.0 * (gc - gh)) / 1024.0
        gs = f16(1024.0 * gc) / 1024.0
        phT, plT = ph.transpose(0, 2, 1), pl.transpose(0, 2, 1)
        ex += phT @ gh
        hgl, lgs = phT @ gl, plT @ gs
        lgh = plT @ gh if "pl_gh" in variants else 0.0
        terms = {"faithful": hgl + lgs, "drop_pl_gs": hgl, "pl_gh": hgl + lgh, "drop_ph_gl": lgs, "no_last_rem": hgl + lgs}
        live = s < nsub
        last = s == nsub - 1
        for v in variants:
            rm[v] += terms[v]
        d1 = np.stack([live & ((((s + mt) % CHAIN) == CHAIN - 1) | last) for mt in range(3)])[tile].T[..., None]
        for v in variants:
            racc[v] = np.where(d1, (racc[v] + ex.astype(np.float32)), racc[v])
        for v in variants:
            end2 = ((s + np.arange(3)) % CHAIN2) == CHAIN2 - 1
            d2 = np.stack([live & (end2[mt] | (last & (v != "no_last_rem"))) for mt in range(3)])[tile].T[..., None]
            racc[v] = np.where(d2, racc[v] + rm[v].astype(np.float32), racc[v])
            rm[v] = np.where(d2, 0.0, rm[v])
        ex = np.where(d1, 0.0, ex)
    fac = np.concatenate([[1.0], scale, scale[P[:, 0]] * scale[P[:, 1]]])
    out = {v: (racc[v].astype(np.float64).sum(0) * fac[:, None]).T for v in variants}
    return out, shift, zb


def np_gamma(x, K, iters=2):
    """Responsibilities [K][N] (float32) of a numpy float64 EM: evenly spaced seed events, global covariance, `iters`
    iterations, then one more E-step."""
    xd = x.astype(np.float64)
    N, D = xd.shape
    mu = xd[np.linspace(0, N - 1, K).astype(np.int64)]
    cov0 = np.cov(xd.T, bias=True).reshape(D, D) + 1e-6 * np.eye(D)
    R = np.repeat(cov0[None], K, 0)
    pi = np.full(K, 1.0 / K)

    def estep():
        ll = np.empty((K, N))
        for k in range(K):
            L = np.linalg.cholesky(R[k])
            y = np.linalg.solve(L, (xd - mu[k]).T)
            ll[k] = np.log(pi[k]) - np.log(np.diag(L)).sum() - 0.5 * (y * y).sum(0)
        ll -= ll.max(0)
        e = np.exp(ll)
        return e / e.sum(0)

    for _ in range(iters):
        gm = estep()
        Nk = gm.sum(1) + 1e-12
        pi = Nk / N
        mu = (gm @ xd) / Nk[:, None]
        for k in range(K):
            y = xd - mu[k]
            R[k] = (gm[k][:, None] * y).T @ y / Nk[k] + 1e-3 * np.diag(np.diag(cov0))
    return estep().astype(np.float32)


def blobs(N, D, K_true, seed):
    return entry.load_package().synth.make_blobs(N, D, K_true, seed=seed)


def outlier_blobs(N, D, ztarget, seed):
    """make_blobs data with one event moved along dimension 0 until its |z| is `ztarget` (the kernel's arithmetic)."""
    x = blobs(N, D, 8, seed).copy()
    for _ in range(4):                                 # the outlier moves the mean and the variance: a few fixed-point steps
        shift, scale, z, _ = standardise(x)
        x[0, 0] = np.float32(shift[0] + ztarget * scale[0])
    return x


# Shapes of tests/test_gpu_mstep_tc.py: every compiled D at K <= 32 and K > 64, the shard and tile edges at D = 12 / 24,
# and the fixed-point range boundary (largest |z| just under 64: zb = 64).
EVERY_D = [(20_000, D, K) for D in (4, 8, 12, 16, 20, 24) for K in (7, 33, 100)]
EDGE_N = [31, 127, 4_095, 4_225, 21_103, 300_001]
EDGES = [(N, D, 8) for D in (12, 24) for N in EDGE_N]


def shape_data(N, D, K):
    x = blobs(N, D, min(K, 16), seed=600 + D)
    return x, np_gamma(x, K)


def model_errors(x, g, variants=VARIANTS):
    """Per-variant worst errors (N, means, R, and the worst of them divided by its bar), and zb."""
    K = g.shape[0]
    emu, shift, zb = emulate(x, g, variants=variants)
    ref = exact_mstep_stats(x, g, shift)
    return {v: mstep_errors(emu[v], ref, shift, K) for v in variants}, zb


_cache = {}


def shape_result(N, D, K):
    key = (N, D, K)
    if key not in _cache:
        x, g = shape_data(N, D, K)
        _cache[key] = model_errors(x, g)
    return _cache[key]


def _fmt(name, e):
    return f"{name:12s} N {e['N']:.2e}  mean {e['mean']:.2e}  R {e['R']:.2e}  (x bar: {e['worst']:.3f})"


ALL = EVERY_D + EDGES


@pytest.mark.parametrize("N,D,K", ALL)
def test_faithful_scheme_within_quarter_bar(N, D, K):
    errs, zb = shape_result(N, D, K)
    print(f"\nN={N} D={D} K={K} zb={zb:g} bar N {MSTEP_TOL['N']:.1e} mean {MSTEP_TOL['mean']:.1e} R {MSTEP_TOL['R']:.1e}")
    for v in VARIANTS:
        print("  " + _fmt(v, errs[v]))
    assert errs["faithful"]["worst"] <= 0.25, errs["faithful"]


def test_faithful_scheme_at_zb64_within_quarter_bar():
    """The worst legal range: one event just under 64 standard deviations (zb = 64) holds the same bar."""
    x = outlier_blobs(200_000, 12, 63.0, seed=611)
    g = np_gamma(x, 8)
    errs, zb = model_errors(x, g, variants=("faithful",))
    print(f"\nzb={zb:g}: " + _fmt("faithful", errs["faithful"]))
    assert zb == 64.0
    assert errs["faithful"]["worst"] <= 0.25, errs["faithful"]


def test_each_kernel_fault_exceeds_the_bar():
    worst = {v: max(shape_result(*s)[0][v]["worst"] for s in ALL) for v in VARIANTS}
    print("\nworst error / bar over the shapes: " + ", ".join(f"{v} {w:.3g}" for v, w in worst.items()))
    for v in ("drop_pl_gs", "pl_gh", "drop_ph_gl", "no_last_rem"):
        assert worst[v] > 1.0, (v, worst[v])


if __name__ == "__main__":
    for s in ALL:
        errs, zb = shape_result(*s)
        print(f"N={s[0]} D={s[1]} K={s[2]} zb={zb:g}")
        for v in VARIANTS:
            print("  " + _fmt(v, errs[v]))
