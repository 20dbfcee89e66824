"""Error model of the tensor E-step (`estep_tc_kernel<D>`, csrc/kernels_tc.cu), on the CPU: the emulation is numpy only
(the parameter sets come from the project's builders and the CPU oracle).

The emulator restates the kernel's operands bit for bit from the parameter set and the context's centre and scale:
  * bimg_cluster(): the Cholesky Gc of the symmetrised Rinv in double (right-looking, as the host code), the rows
    W'[d][j] = fl32(Gc[j][d] * scale_j), v_d = the fma chain -sum_j Gc[j][d] (mu_j - s_j), the per-cluster power of two
    e2 = 12 - ilogb(amax) clamped to +-40, Wh / Wl = the FP16 round-to-nearest split of 2^e2 W', vh / vl that of 2^e2 v;
  * the constants: ck = constant + fl32(ln pi in double), the kernel's fl32(ck * log2 e), and the multiplier
    fl32(-1/2 log2 e 4^-e2);
  * z = fl32(fl32(x - s) * inv_scale) and its hi / lo split (tc_split_rows).
y is then the float64 sum of exactly the products the kernel keeps, zh Wh + zl Wh + zh Wl + vh + vl over the
block-triangular chunks, squared and summed, turned into the base-2 logits, and the log-sum-exp is taken in float64.
What is not emulated is the tensor cores' FP32 accumulation and the epilogue's FP32 / ex2.approx / logf rounding.

The bar (estep_bar) bounds, per (event, cluster), what is not emulated:
  * the FP32 accumulation of the wgmma k-steps.  Assumed truncating, as the M-step's model assumes (DESIGN 5.2): every
    k-step of output column d's block c may lose 1 ulp (2^-23 relative) of a running sum bounded by sum_j |terms|, so
    |dy_d| <= nk_c 2^-23 sum|terms_d|, nk_c = (CP - c) + ceil((CP - c + 1) / 2) k-steps;
  * the FP32 square-and-sum (2 CP fmas and 2 shuffle adds of positive terms: (2 CP + 3) u relative, u = 2^-24) and the
    rounding of the logit fma (u |l|);
  * the subtraction l - M (u |l - M|), ex2.approx.ftz.f32 (PTX ISA: at most 2 ulp, 2^-22 relative), the FP32 sums of the
    denominator ((4 NSG + 2) u), the IEEE 1/S and the final product (u each); at K > 64 the join of the passes' log-
    denominators (__expf: 2 + 1.173 |x| ulp, logf, and the base-2 conversion of the total).
Per cluster with r_k = ln2 (dl_k + u |l_k - M|) + 2^-22 and rho = sum_j gamma_j (e^(r_j) - 1):
    |gamma_gpu - gamma_emu| <= gamma_emu max(e^(r_k) (1+u)^2 / ((1-rho)(1-s)) - 1,  1 - e^(-r_k) (1-u)^2 / ((1+rho)(1+s)))
                               + 2^-122   (the flush-to-zero region: below 2^-126 a responsibility may be 0).
The log-density is held to |logp_gpu - lse_emu| <= rho + s + 2^-22 (|lse| + |M ln2| + 1) (+ the join at K > 64).

The module asserts, on the parameter sets and (D, K) of tests/test_gpu_estep_tc.py:
  1. a faithful FP32 emulation (round-to-nearest and truncating k-step accumulation in the kernel's order, the fma
     square-and-sum with the quad transpose, the epilogue's FP32 operations and summation order) stays at or below a
     quarter of the bar;
  2. each of these kernel faults exceeds the bar at one shape at least: the zl Wh product dropped, the zh Wl product
     dropped, vl dropped, the logits of two clusters of one 4-cluster chunk swapped (a logit slot read with another
     event's swizzle; this fault passes the per-operator 1e-4 / 1e-6 bar of tests/test_gpu_parity.py), and a wrong
     per-cluster 4^-e2 (cluster k scaled with cluster k ^ 1's);
  3. the emulated y stays within the bound of the dropped lo * lo product (and the FP16 / FP32 roundings of the lo
     parts) of a float64 evaluation with the unsplit double factor, so the emulator models the same mathematics;
  4. with components at pi = 0 (ck = -inf; one ahead of the others, one alone in the last pass, a whole pass) the
     emulation gives them gamma = 0 exactly and the log-sum-exp of the others, and the faithful epilogue stays within a
     quarter of the bar.
  5. the scoring epilogue (fp32_score) on SCORE_SHAPES: faithful within a quarter of the bars (max_resp against gbar of
     its label, logp against lbar, no sure label differing) and max_resp equal to fp32_gamma's value of the label; each of
     SCORE_FAULTS fails at one shape at least (a later pass winning ties, kbase dropped, an earlier winner with the current
     pass's M and S, the __expf(den - tot) factor dropped, a pass left out of the join).
The shapes include D = 8, whose fused epilogue (estep_fused) forms the split epilogue's values (fp32_gamma); every fault
exceeds the bar at a D = 8 shape.
Run it as a script (python tests/test_estep_error_model.py) for the table of worst error / bar per shape.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import entry, fitted_params, random_spd_params  # noqa: E402
from test_mstep_error_model import f16, f32, standardise  # noqa: E402

U = 2.0 ** -24
LOG2E, LN2 = 1.4426950408889634, 0.6931471805599453
LOG2E_F, LN2_F = float(np.float32(LOG2E)), float(np.float32(LN2))
FTZ = 2.0 ** -126
FLT_MAX = float(np.finfo(np.float32).max)
FTZ_SLACK = 2.0 ** -122   # absolute slack of the bar: a responsibility (or a term of the denominator) below 2^-126 may be 0
VARIANTS = ("faithful_rn", "faithful_trunc", "drop_zl_wh", "drop_zh_wl", "drop_vl", "chunk_swap", "wrong_e2")
FAULTS = VARIANTS[2:]


# ---- operands (bimg_cluster, tc_split_rows) -------------------------------------------------------------------------
def _fma(a, b, c):
    """fl64(a * b + c) with the product exact (Dekker), as std::fma up to a rare last-bit tie."""
    a, b, c = (np.asarray(t, np.float64) for t in (a, b, c))
    p = a * b
    sp = 134217729.0
    ah = a * sp - (a * sp - a)
    bh = b * sp - (b * sp - b)
    pl = ((ah * bh - p) + ah * (b - bh) + (a - ah) * bh) + (a - ah) * (b - bh)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    return s + (e + pl)


def operands(cl, K, shift, scale):
    """Per cluster k < K: Wh, Wl [K][D][D] (FP16 values, scaled by 2^e2, upper triangular), vh, vl [K][D], e2 [K],
    the logit constant ck_s = fl32(ck * log2 e) and multiplier mult [K] as float64 values of the kernel's floats, and
    the unsplit double factor Wx = 2^e2 W' (exact product, before the FP32 rounding) and vx = 2^e2 v."""
    D = cl.means.shape[1]
    Ri = cl.Rinv[:K].astype(np.float64)
    A = 0.5 * (Ri + Ri.transpose(0, 2, 1))
    G = np.zeros((K, D, D))
    for j in range(D):                                     # right-looking Cholesky A = G G^T
        piv = np.sqrt(A[:, j, j])
        G[:, j, j] = piv
        G[:, j + 1:, j] = A[:, j + 1:, j] * (1.0 / piv)[:, None]
        l = G[:, j + 1:, j]
        A[:, j + 1:, j + 1:] -= l[:, :, None] * l[:, None, :]
    Wd = np.triu(G.transpose(0, 2, 1))                    # W[d][j] = G[j][d], j >= d
    Wx = Wd * scale[None, None, :]
    wrow = f32(Wx)
    dm = cl.means[:K].astype(np.float64) - shift[None, :]
    v = np.zeros((K, D))
    for j in range(D):
        v = _fma(-Wd[:, :, j], dm[:, j][:, None], v)
    amax = np.maximum(np.abs(wrow).max((1, 2)), f32(np.abs(v)).max(1))
    e2 = np.where(amax > 0, 12 - (np.frexp(amax)[1] - 1), 0)
    e2 = np.clip(e2, -40, 40)
    sc = np.ldexp(1.0, e2)[:, None, None]
    wrow = f32(wrow * sc)
    Wh = f16(wrow)
    Wl = f16(f32(wrow - Wh))
    vs = v * sc[:, :, 0]
    vh = f16(f32(vs))
    vl = f16(f32(vs - vh))
    ck = f32(cl.constant[:K].astype(np.float64) + f32(np.log(cl.pi[:K].astype(np.float64))))
    ck_s = f32(ck * LOG2E_F)
    mult = f32(np.ldexp(-0.5 * LOG2E, -2 * e2))
    return dict(Wh=Wh, Wl=Wl, vh=vh, vl=vl, e2=e2, ck=ck_s, mult=mult, Wx=Wx * sc, vx=vs)


def split_events(x, shift, scale):
    """z, zh, zl [N][D] as tc_split_rows forms them (float64 values of the kernel's floats / halves)."""
    sf = shift.astype(np.float32)
    isf = (1.0 / scale).astype(np.float32)
    z = ((np.asarray(x, np.float32) - sf) * isf).astype(np.float64)
    zh = f16(z)
    return z, zh, f16(f32(z - zh))


def nk_of_column(D):
    """k-steps of the block of each output column (tc_issue_group)."""
    CP = D // 8
    c = np.arange(D) // 8
    return (CP - c) + (CP - c + 2) // 2


# ---- emulation ----------------------------------------------------------------------------------------------------------
def kept_y(op, zh, zl, drop=()):
    """y [N][K][D] = the float64 sum of the kept products, and sum |terms| per output."""
    K, D = op["vh"].shape
    W1 = op["Wh"] + (0.0 if "zh_wl" in drop else op["Wl"])
    y = (zh @ W1.reshape(K * D, D).T).reshape(-1, K, D)
    if "zl_wh" not in drop:
        y += (zl @ op["Wh"].reshape(K * D, D).T).reshape(-1, K, D)
    y += op["vh"][None] + (0.0 if "vl" in drop else op["vl"][None])
    T = (np.abs(zh) @ (np.abs(op["Wh"]) + np.abs(op["Wl"])).reshape(K * D, D).T + np.abs(zl) @ np.abs(op["Wh"]).reshape(K * D, D).T)
    T = T.reshape(-1, K, D) + np.abs(op["vh"])[None] + np.abs(op["vl"])[None]
    return y, T


def _round32(a, trunc):
    r = a.astype(np.float32)
    if trunc:
        over = np.abs(r.astype(np.float64)) > np.abs(a)
        r = np.where(over, np.nextafter(r, np.float32(0)), r)
    return r.astype(np.float64)


def fp32_y(op, zh, zl, trunc):
    """y with the kernel's k-steps (tc_issue_group) each added to an FP32 accumulator, rounded to nearest or truncated."""
    K, D = op["vh"].shape
    CP = D // 8
    N = zh.shape[0]
    y = np.empty((N, K, D))
    ones = np.zeros((N, 8))
    ones[:, :2] = 1.0
    vchunk = np.zeros((K, D, 8))
    vchunk[:, :, 0], vchunk[:, :, 1] = op["vh"], op["vl"]
    for c in range(CP):
        cols = slice(8 * c, 8 * c + 8)
        steps = [[(zh[:, 8 * j:8 * j + 8], op["Wh"][:, cols, 8 * j:8 * j + 8]), (zh[:, 8 * j:8 * j + 8], op["Wl"][:, cols, 8 * j:8 * j + 8])]
                 for j in range(c, CP)]
        for p in range(c, CP + 1, 2):
            x_, y_ = p, p + 1
            if y_ <= CP:
                second = (zl[:, 8 * y_:8 * y_ + 8], op["Wh"][:, cols, 8 * y_:8 * y_ + 8]) if y_ < CP else (ones, vchunk[:, cols])
                steps.append([(zl[:, 8 * x_:8 * x_ + 8], op["Wh"][:, cols, 8 * x_:8 * x_ + 8]), second])
            else:
                steps.append([(ones, vchunk[:, cols])])
        acc = np.zeros((N, K * 8))
        for st in steps:
            part = sum(a @ b.reshape(K * 8, 8).T for a, b in st)
            acc = _round32(acc + part, trunc)
        y[:, :, cols] = acc.reshape(N, K, 8)
    return y


def fp32_logits(op, y):
    """The square-and-sum (two columns per quad lane, fma chain over the blocks, then the quad transpose) and the logit fma."""
    N, K, D = y.shape
    CP = D // 8
    s = []
    for q in range(4):
        a = np.zeros((N, K))
        for c in range(CP):
            y0, y1 = y[:, :, 8 * c + 2 * q], y[:, :, 8 * c + 2 * q + 1]
            a = f32(y0 * y0 + f32(y1 * y1 + a))
        s.append(a)
    qv = f32(f32(s[0] + s[1]) + f32(s[2] + s[3]))
    return f32(op["mult"][None] * qv + op["ck"][None])


def _ex2(a):
    t = f32(np.exp2(a))
    return np.where(t < FTZ, 0.0, t)


def fp32_gamma(l, K):
    """The split epilogue's FP32 operations per 64-cluster pass and, at K > 64, the join of the passes (modes 1, 2, 3).
    The fused D = 8 epilogue (estep_fused) forms the same values: its lane qd sums the 4-cluster chunk 4 sg + cq of every
    supergroup (cq = 0, 2, 1, 3 for qd = 0 .. 3) in (supergroup, cluster) order, starting from 0 and adding the exact 0 of
    the supergroups past NSG; the two quad shuffles then give (P0 + P1) + (P2 + P3) on every lane (each addition is
    commutative), which is a0 + a1 below with a_hh = p0 + p1 over the chunks hh and 2 + hh.  Its 1 / S, the join and the
    mode 3 subtrahend fl32(tot * log2 e) (an FMUL of its own in the SASS, not contracted into the subtraction) are the
    split kernel's operations.  Both start the maximum at -FLT_MAX: a pass without a finite logit (every pi 0) has S = 0,
    a log-denominator of -inf and responsibilities of 0."""
    passes, t_all, den, S_all, M_all = fp32_passes(l, K)
    if len(passes) == 1:
        g = f32(t_all[0] * f32(1.0 / S_all[0])[:, None])
        return np.where(np.abs(g) < FTZ, 0.0, g), den[0]
    tot = fp32_join(den)
    out = []
    sub = f32(tot * LOG2E_F)
    for p, (k0, k1) in enumerate(passes):
        if p == len(passes) - 1:
            with np.errstate(divide="ignore", invalid="ignore"):
                scl = np.where(S_all[p] == 0, 0.0, f32(f32(1.0 / S_all[p]) * f32(np.exp(den[p] - tot))))
            g = f32(t_all[p] * scl[:, None])
        else:
            g = _ex2(f32(l[:, k0:k1] - sub[:, None]))
        out.append(np.where(np.abs(g) < FTZ, 0.0, g))
    return np.concatenate(out, 1), tot


PAD_L2 = float(np.float32(np.float32(-1e30) * np.float32(LOG2E_F)))   # a padding cluster's logit: ck = -1e30, multiplier 0


def fp32_passes(l, K):
    """Per 64-cluster pass: (k0, k1), the terms ex2(l - M) of its clusters, its log-denominator, S and M, with the
    epilogue's FP32 operations.  The pass's padding clusters (up to a multiple of 16, tc_params_begin) are in M and S: their
    logit is PAD_L2, so they add 0 unless no cluster of the pass has a finite logit (then S counts them); M starts at
    -FLT_MAX, so a pass of 16 n clusters without a finite logit has S = 0 and a log-denominator of -inf."""
    N = l.shape[0]
    passes = [(p * 64, min(K, p * 64 + 64)) for p in range((K + 63) // 64)]
    t_all, den, S_all, M_all = [], [], [], []
    for k0, k1 in passes:
        Kp = k1 - k0
        nsg = (Kp + 15) // 16
        lp = np.concatenate([l[:, k0:k1], np.full((N, nsg * 16 - Kp), PAD_L2)], 1)
        M = np.maximum(lp.max(1), -FLT_MAX)
        tt = _ex2(f32(lp - M[:, None]))
        t = tt[:, :Kp]
        a = []
        for hh in range(2):
            p0 = np.zeros(N)
            p1 = np.zeros(N)
            for sg in range(nsg):
                for i in range(4):
                    p0 = f32(p0 + tt[:, 16 * sg + 4 * hh + i])
                for i in range(4):
                    p1 = f32(p1 + tt[:, 16 * sg + 8 + 4 * hh + i])
            a.append(f32(p0 + p1))
        S = f32(a[0] + a[1])
        with np.errstate(divide="ignore"):
            den.append(f32(M * LN2_F + f32(np.log(S))))
        t_all.append(t)
        S_all.append(S)
        M_all.append(M)
    return passes, t_all, den, S_all, M_all


def join1(d, run):
    """One join of a pass's log-denominator d with the running one (E-step modes 1 / 2, score_tc_kernel)."""
    gm = np.maximum(np.maximum(d, run), -FLT_MAX)
    with np.errstate(invalid="ignore"):
        return f32(gm + f32(np.log(f32(f32(np.exp(d - gm)) + f32(np.exp(run - gm))))))


def fp32_join(den):
    tot = den[0]
    for d in den[1:]:
        tot = join1(d, tot)
    return tot


# ---- the scoring epilogue (score_tc_kernel) ----------------------------------------------------------------------------------
SCORE_FAULTS = ("later_pass_wins_ties", "kbase_dropped", "earlier_winner_current_pass", "join_factor_dropped", "pass_left_out")


def fp32_score(l, K, fault=None):
    """(labels, max_resp, logp) of score_tc_kernel on the base-2 logits l [N][K], with its FP32 operations.
    Per pass the arg-max runs over the lane's 16 logits in increasing k, then over the quad with (value, index) pairs and
    the lower index on equal values: the first maximum in k order, numpy's argmax.  Across passes the running best is
    replaced only by a strictly larger logit (an earlier pass wins ties), the label is kbase + k.  max_resp at K <= 64 is
    ex2(bl - M) (1 / S); at K > 64 the last pass's winner takes ex2(bl - M) ((1 / S) __expf(den - tot)) (E-step mode 2) and
    an earlier pass's winner ex2(bl - fl(tot log2 e)) (mode 3); logp is the joined log-denominator.  `fault` is one of
    SCORE_FAULTS."""
    N = l.shape[0]
    passes, _, den, S_all, M_all = fp32_passes(l, K)
    rows = np.arange(N)
    rbl = rbk = rden = None
    for p, (k0, k1) in enumerate(passes):
        lp = l[:, k0:k1]
        idx = np.argmax(lp, 1)
        bl = lp[rows, idx]
        bk = idx + (0 if fault == "kbase_dropped" else k0)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv_s = f32(1.0 / S_all[p])
        if p == 0:
            rbl, rbk, rden = bl, bk, den[0]
            mr = f32(_ex2(f32(bl - M_all[0])) * inv_s)
            continue
        tot = den[p] if (fault == "pass_left_out" and p == 1) else join1(den[p], rden)
        wins = bl >= rbl if fault == "later_pass_wins_ties" else bl > rbl
        with np.errstate(invalid="ignore"):
            sc = inv_s if fault == "join_factor_dropped" else f32(inv_s * f32(np.exp(den[p] - tot)))
        mine = f32(_ex2(f32(bl - M_all[p])) * sc)
        if fault == "earlier_winner_current_pass":
            theirs = f32(_ex2(f32(rbl - M_all[p])) * f32(inv_s * f32(np.exp(den[p] - tot))))
        else:
            theirs = _ex2(f32(rbl - f32(tot * LOG2E_F)))
        mr = np.where(wins, mine, theirs)
        rbl, rbk, rden = np.where(wins, bl, rbl), np.where(wins, bk, rbk), tot
    return rbk, np.where(np.abs(mr) < FTZ, 0.0, mr), rden


def logits64(op, y):
    return op["mult"][None] * (y * y).sum(2) + op["ck"][None]


def lse2(l):
    """gamma and the natural log-sum-exp of base-2 logits [N][K], in float64 (-inf, and gamma 0, where no logit is finite)."""
    M = np.maximum(l.max(1), -FLT_MAX)
    t = np.exp2(l - M[:, None])
    S = t.sum(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(S[:, None] > 0, t / S[:, None], 0.0), (M + np.log2(S)) * LN2


# ---- the bar --------------------------------------------------------------------------------------------------------------
def estep_bar(op, y, T, l, gamma, lse):
    """Per-(event, cluster) bound on |gamma_gpu - gamma_emu| and per-event bound on |logp_gpu - lse_emu| (module docstring)."""
    N, K, D = y.shape
    CP = D // 8
    E = nk_of_column(D)[None, None, :] * 2.0 ** -23 * T
    qv = (y * y).sum(2)
    dqv = (2 * np.abs(y) * E + E * E).sum(2) + (2 * CP + 3) * U * qv
    dl = np.abs(op["mult"])[None] * dqv + U * np.abs(l)
    M = np.maximum(l.max(1), -FLT_MAX)
    r = LN2 * (dl + U * np.abs(l - M[:, None])) + 2.0 ** -22
    multi = K > 64
    if multi:                                              # the join of the passes' log-denominators and its base-2 conversion
        den_p = np.empty((N, K))
        for k0 in range(0, K, 64):
            den_p[:, k0:k0 + 64] = lse2(l[:, k0:k0 + 64])[1][:, None]
        r = r + (2.0 + 1.173 * np.abs(den_p - lse[:, None])) * 2.0 ** -23 + 2.0 ** -20 * (1.0 + np.abs(lse))[:, None]
    r = np.minimum(r, 700.0)                              # (clusters that far away have gamma = 0)
    live = gamma > 0
    rho = np.where(live, gamma * np.expm1(r), 0.0).sum(1)
    s = (20 if multi else 4 * ((K + 15) // 16) + 2) * U
    hi = np.exp(r) * (1 + U) ** 2 / ((1 - rho) * (1 - s))[:, None] - 1
    lo = 1 - np.exp(-r) * (1 - U) ** 2 / ((1 + rho) * (1 + s))[:, None]
    gbar = np.where(live, gamma * np.maximum(hi, lo), 0.0) + FTZ_SLACK
    # rho >= 1 (logits off by about an ulp of a logit near 2^23 or more, e.g. events 2^10 standard deviations out): the
    # model bounds no responsibility of the event (it would give a negative bar), only its log-density
    gbar = np.where((rho < 1.0)[:, None], gbar, np.inf)
    lbar = rho + s + 2.0 ** -22 * (np.abs(lse) + np.abs(M * LN2) + 1.0)
    if multi:
        lbar = lbar + 2.0 ** -20 * (1.0 + np.abs(lse))
    return gbar, lbar, dl


class Emulation:
    """The emulated responsibilities, log-densities and their bars for events x under the parameter set cl."""

    def __init__(self, cl, K, x, shift, scale):
        self.K = K
        self.op = operands(cl, K, shift, scale)
        self.z, self.zh, self.zl = split_events(x, shift, scale)
        self.y, self.T = kept_y(self.op, self.zh, self.zl)
        self.l = logits64(self.op, self.y)
        self.gamma, self.lse = lse2(self.l)
        self.gbar, self.lbar, self.dl = estep_bar(self.op, self.y, self.T, self.l, self.gamma, self.lse)

    def ratio(self, gamma):
        """Worst |gamma - gamma_emu| / bar over all events and clusters; gamma is [K][N] or [N][K]."""
        g = np.asarray(gamma, np.float64)
        if g.shape != self.gamma.shape:
            g = g.T
        return float((np.abs(g - self.gamma) / self.gbar).max())

    def lse_ratio(self, logp):
        d = np.abs(np.asarray(logp, np.float64) - self.lse) / self.lbar
        return float(np.where(np.isnan(d), np.inf, d).max())

    def score_check(self, labels, max_resp, logp):
        """gmm_score's outputs against the emulation: (worst |max_resp - gamma_emu[label]| / gbar[label], worst
        |logp - lse| / lbar, events whose label differs from the emulated arg-max where that label is sure).  A label is
        sure where the emulated top-two gap exceeds both logits' bars (dl, base 2), or where the top logits are exactly
        equal (identical operands, identical FP32 logits: the lowest k wins)."""
        lab = np.asarray(labels)
        rows = np.arange(len(lab))
        mr = np.asarray(max_resp, np.float64)
        d = np.abs(mr - self.gamma[rows, lab]) / self.gbar[rows, lab]
        r_mr = float(np.where(np.isnan(d), np.inf, d).max())      # a NaN max_resp fails
        r_lp = self.lse_ratio(logp)
        order = np.argsort(-self.l, axis=1, kind="stable")
        top, second = order[:, 0], order[:, 1] if self.K > 1 else order[:, 0]
        gap = self.l[rows, top] - self.l[rows, second]
        sure = (gap > self.dl[rows, top] + self.dl[rows, second]) | (gap == 0) if self.K > 1 else np.ones(len(lab), bool)
        return r_mr, r_lp, int((sure & (lab != top)).sum())

    def old_bar_passes(self, gamma):
        g = np.asarray(gamma, np.float64)
        return bool((np.abs(g - self.gamma) <= 1e-4 * np.abs(self.gamma) + 1e-6).all())


def variant_gamma(em, v):
    """Responsibilities [N][K] of the kernel variant v (faithful FP32 emulations, or a fault on the float64 emulation)."""
    op, K = em.op, em.K
    if v.startswith("faithful"):
        y = fp32_y(op, em.zh, em.zl, trunc=v.endswith("trunc"))
        return fp32_gamma(fp32_logits(op, y), K)[0]
    if v.startswith("drop"):
        y, _ = kept_y(op, em.zh, em.zl, drop=(v[5:],))
        return lse2(logits64(op, y))[0]
    if v == "wrong_e2":
        o2 = dict(op)
        o2["mult"] = op["mult"][np.minimum(np.arange(K) ^ 1, K - 1)]
        return lse2(logits64(o2, em.y))[0]
    if v == "chunk_swap":
        a, b = swap_pair(em)
        l = em.l.copy()
        l[:, [a, b]] = l[:, [b, a]]
        return lse2(l)[0]
    raise ValueError(v)


def swap_pair(em):
    """Two clusters of one 4-cluster chunk with the smallest responsibilities over the events (the swap the per-operator
    bar cannot see)."""
    K = em.K
    top = em.gamma.max(0)
    best = None
    for c in range((K + 3) // 4):
        ks = [k for k in range(4 * c, min(K, 4 * c + 4))]
        for i in range(len(ks)):
            for j in range(i + 1, len(ks)):
                w = max(top[ks[i]], top[ks[j]])
                if best is None or w < best[0]:
                    best = (w, ks[i], ks[j])
    return (best[1], best[2]) if best else (0, 0)


def oracle_y_ratio(em):
    """Worst |y_emu - y64| over the bound of what the split drops (lo * lo, and the FP16 / FP32 roundings of the lo parts
    and of W', whose FP16 subnormals hold 2^-25 absolute): y64 = 2^e2 (W' z + v) from the unsplit double factor on the
    same float32 z."""
    op = em.op
    K, D = op["vh"].shape
    y64 = (em.z @ op["Wx"].reshape(K * D, D).T).reshape(-1, K, D) + op["vx"][None]
    S = (np.abs(em.z) @ np.abs(op["Wx"]).reshape(K * D, D).T).reshape(-1, K, D) + np.abs(op["vx"])[None]
    sub = np.abs(op["Wx"]).sum(2)[None] + np.abs(em.z).sum(1)[:, None, None] + 1.0
    bound = 2.0 ** -20 * S + 2.0 ** -24 * sub
    return float((np.abs(em.y - y64) / bound).max())


# ---- parameter sets and shapes (shared with tests/test_gpu_estep_tc.py) ---------------------------------------------------
KINDS = ("fitted", "spd", "needle")
ERR_D = (8, 16, 24)
ERR_K = (17, 64, 129)
N_FIT = 20_000
N_DATA = 480_000          # the deep shapes of the GPU test use a prefix of these events


def blobs(D):
    """The events of the GPU test at this D: 16 blobs, N_DATA events (parameters are fitted on the first N_FIT)."""
    return entry.load_package().synth.make_blobs(N_DATA, D, 16, seed=700 + D)


def param_set(pkg, oracle, kind, D, K, ev):
    """fitted: the oracle's seeding + 2 EM iterations on the first 20 000 events; spd: random_spd_params (spread 6,
    Mahalanobis distances of several hundred); needle: fitted, with two needle clusters (sigma 1e-4) sitting on events
    and one cluster far wider than the data (extreme e2 both ways)."""
    if kind == "spd":
        cl = random_spd_params(pkg, K, D, np.random.default_rng(D * 7 + K), spread=6.0)
        oracle.constants(cl, K)
        return cl
    cl = fitted_params(pkg, oracle, np.ascontiguousarray(ev[:N_FIT]), K)
    if kind == "needle":
        rng = np.random.default_rng(K)
        for k, idx in ((0, 123), (K - 1, 4567)):
            cl.means[k] = ev[idx] + rng.normal(0, 1e-4, D).astype(np.float32)
            cl.R[k] = np.eye(D, dtype=np.float32) * np.float32(1e-8)
            cl.N[k] = 3.0
        cl.R[1] = np.eye(D, dtype=np.float32) * np.float32(400.0)
        oracle.constants(cl, K)
    return cl


N_CPU = 3_000
SHAPES = [(kind, D, K) for kind in KINDS for D in ERR_D for K in ERR_K]

_cache = {}


def shape_result(kind, D, K):
    key = (kind, D, K)
    if key not in _cache:
        pkg = entry.load_package()
        oracle = entry.load_oracle("f64")
        ev = blobs(D)
        cl = param_set(pkg, oracle, kind, D, K, ev)
        shift, scale = standardise(ev)[:2]
        idx = np.r_[np.arange(N_CPU - 2), 123, 4567]                  # the needles' events too
        em = Emulation(cl, K, ev[idx], shift, scale)
        res = {}
        for v in VARIANTS:
            g = variant_gamma(em, v)
            res[v] = em.ratio(g)
            if v == "chunk_swap":
                res["chunk_swap_old_bar_passes"] = em.old_bar_passes(g)
        res["oracle_y"] = oracle_y_ratio(em)
        res["e2"] = (int(em.op["e2"].min()), int(em.op["e2"].max()))
        _cache[key] = res
    return _cache[key]


def _fmt(key, r):
    return (f"{key[0]:6s} D={key[1]} K={key[2]:3d} e2 {r['e2'][0]:+d}..{r['e2'][1]:+d}  " + "  ".join(f"{v} {r[v]:.3g}" for v in VARIANTS)
            + f"  (swap passes old bar: {r['chunk_swap_old_bar_passes']})  y vs f64 {r['oracle_y']:.3g}")


@pytest.mark.parametrize("kind,D,K", SHAPES)
def test_faithful_fp32_within_quarter_bar(kind, D, K):
    r = shape_result(kind, D, K)
    print("\n" + _fmt((kind, D, K), r))
    assert r["faithful_rn"] <= 0.25 and r["faithful_trunc"] <= 0.25, r
    assert r["oracle_y"] <= 1.0, r


def test_each_kernel_fault_exceeds_the_bar():
    res = {s: shape_result(*s) for s in SHAPES}
    worst = {v: max(r[v] for r in res.values()) for v in FAULTS}
    print("\nworst error / bar over the shapes: " + ", ".join(f"{v} {w:.3g}" for v, w in worst.items()))
    for v in FAULTS:
        assert worst[v] > 1.0, (v, worst[v])
    # a chunk swap the per-operator bar (1e-4 relative, 1e-6 absolute) passes, and this bar does not
    assert any(r["chunk_swap"] > 1.0 and r["chunk_swap_old_bar_passes"] for r in res.values())


# ---- the scoring epilogue: shapes, faithful emulation and faults ------------------------------------------------------------
SCORE_SHAPES = [(kind, D, K) for kind in ("fitted", "spd") for D in ERR_D for K in (7, 65, 129)] + [("dup", D, 129) for D in ERR_D]
_score_cache = {}


def score_shape(kind, D, K):
    """Emulation and score outputs on N_CPU events: "dup" is the fitted set with cluster k + 64 a copy of cluster k."""
    key = (kind, D, K)
    if key not in _score_cache:
        pkg = entry.load_package()
        oracle = entry.load_oracle("f64")
        ev = blobs(D)
        cl = param_set(pkg, oracle, "fitted" if kind == "dup" else kind, D, K, ev)
        if kind == "dup":
            for f in ("means", "R", "Rinv", "constant", "pi", "N"):
                getattr(cl, f)[64:128] = getattr(cl, f)[0:64]
        shift, scale = standardise(ev)[:2]
        em = Emulation(cl, K, ev[:N_CPU], shift, scale)
        res = {}
        for trunc in (False, True):
            l32 = fp32_logits(em.op, fp32_y(em.op, em.zh, em.zl, trunc=trunc))
            lab, mr, lp = fp32_score(l32, K)
            g = fp32_gamma(l32, K)[0]
            res["faithful_" + ("trunc" if trunc else "rn")] = em.score_check(lab, mr, lp)
            # max_resp is the E-step's stored responsibility of the label, bit for bit
            res["identity_" + ("trunc" if trunc else "rn")] = bool(np.array_equal(mr, g[np.arange(len(lab)), lab]))
            if not trunc:
                for v in SCORE_FAULTS:
                    res[v] = em.score_check(*fp32_score(l32, K, fault=v))
        _score_cache[key] = res
    return _score_cache[key]


@pytest.mark.parametrize("kind,D,K", SCORE_SHAPES)
def test_score_faithful_within_quarter_bar(kind, D, K):
    r = score_shape(kind, D, K)
    print(f"\nscore {kind} D={D} K={K}: " + "  ".join(f"{v} {r[v][0]:.3g}/{r[v][1]:.3g}/{r[v][2]}" for v in ("faithful_rn", "faithful_trunc") + SCORE_FAULTS))
    for v in ("faithful_rn", "faithful_trunc"):
        assert r[v][0] <= 0.25 and r[v][1] <= 0.25 and r[v][2] == 0, (v, r[v])
        assert r["identity_" + v[9:]], v


def test_each_scoring_fault_fails():
    """Each fault exceeds the max_resp or the logp bar, or gives a sure label that differs, at some shape."""
    res = {s: score_shape(*s) for s in SCORE_SHAPES}
    for v in SCORE_FAULTS:
        caught = [s for s, r in res.items() if r[v][0] > 1.0 or r[v][1] > 1.0 or r[v][2] > 0]
        print(f"\n  {v}: caught at {len(caught)} of {len(res)} shapes")
        assert caught, v


@pytest.mark.parametrize("D,K,zero", [(8, 17, [0]), (16, 65, [64]), (24, 129, list(range(64))), (8, 130, list(range(64, 128))),
                                      (16, 70, [0, 5, 63]), (8, 80, list(range(64, 80))),
                                      (24, 128, list(range(64, 128)))])
def test_zero_pi_components(D, K, zero):
    """pi = 0: ck = -inf.  The emulation gives those components gamma = 0 exactly and the log-sum-exp of the others, the
    bar is finite, and the faithful FP32 epilogue (a -inf pass maximum floored at -FLT_MAX) stays within a quarter of it."""
    pkg = entry.load_package()
    oracle = entry.load_oracle("f64")
    ev = blobs(D)
    cl = param_set(pkg, oracle, "fitted", D, K, ev)
    cl.pi[zero] = 0.0
    shift, scale = standardise(ev)[:2]
    with np.errstate(divide="ignore"):
        em = Emulation(cl, K, ev[:N_CPU], shift, scale)
    assert np.all(em.op["ck"][zero] == -np.inf) and np.all(em.l[:, zero] == -np.inf)
    for a in (em.gamma, em.lse, em.gbar, em.lbar):
        assert not np.isnan(a).any()
    assert np.all(em.gamma[:, zero] == 0.0) and np.isfinite(em.lse).all()
    keep = np.setdiff1d(np.arange(K), zero)
    np.testing.assert_allclose(em.lse, lse2(em.l[:, keep])[1], rtol=1e-15, atol=0)
    for v in ("faithful_rn", "faithful_trunc"):
        with np.errstate(divide="ignore", invalid="ignore"):
            g = variant_gamma(em, v)
        assert not np.isnan(g).any() and np.all(g[:, zero] == 0.0), v
        assert em.ratio(g) <= 0.25, (v, em.ratio(g))


def test_bar_helpers_on_a_known_case():
    """nk per column, the per-cluster power of two, and the factor: W^T W reproduces the symmetrised Rinv."""
    assert list(nk_of_column(24)[::8]) == [5, 4, 2] and list(nk_of_column(16)[::8]) == [4, 2] and list(nk_of_column(8)) == [2] * 8
    pkg = entry.load_package()
    cl = random_spd_params(pkg, 5, 16, np.random.default_rng(1))
    cl.Rinv[:5] = np.linalg.inv(cl.R[:5].astype(np.float64)).astype(np.float32)
    cl.pi[:5] = 0.2
    op = operands(cl, 5, np.zeros(16), np.ones(16))
    amax = np.maximum(np.abs(f32(op["Wx"])).max((1, 2)), np.abs(op["vx"]).max(1))
    assert np.all((amax >= 2 ** 12) & (amax < 2 ** 13))                   # the largest operand entry in [2^12, 2^13)
    Rinv = cl.Rinv[:5].astype(np.float64)
    Wd = op["Wx"] / np.ldexp(1.0, op["e2"])[:, None, None]
    np.testing.assert_allclose(Wd.transpose(0, 2, 1) @ Wd, 0.5 * (Rinv + Rinv.transpose(0, 2, 1)), rtol=1e-12, atol=1e-12)


if __name__ == "__main__":
    for s in SHAPES:
        print(_fmt(s, shape_result(*s)))
