// kernels_modes.cuh — the mode-finding kernels of gmm_modes / gmm_mode_labels, for sm_90a.
//
// Every point x (an event, or a component mean for gmm_modes) climbs ln p(x) = ln sum_k exp l_k(x) by the fixed point of
// Carreira-Perpinan (2000) in step form (the semantics are spelt out in gmm.h):
//   dx_k = x - mu_k,  l_k = const_k - dx_k^T S_k dx_k / 2,  r_k = exp(l_k - ln p),
//   g = sum_k r_k S_k (-dx_k),  A = sum_k r_k S_k,  delta = A^-1 g (Cholesky),  x <- x + delta.
// The modes are the points with g = 0 whatever A is: A's rounding changes how fast a point converges, never where.
// Coordinates are relative to the host's float centre c.  Component records (mode_rec_floats(DP) floats each, DP = D rounded
// up to a multiple of 4, the component count padded to a multiple of kModeChunk with inert records):
//   [ mu~ (DP) | S = (P + P^T) / 2 row-major (DP x DP) | const + ln pi | 3 zeros ],  zero beyond D.
// An inert record has mu~ = S = 0 and const = -inf: its logit is -inf, its weight exactly 0, and every sum it enters keeps
// its bits.  Padded dimensions are inert too: x = mu~ = 0 there, S has zero rows and columns, and A gets a unit diagonal,
// so delta = 0 on them.
#pragma once
#include <cuda_runtime.h>
#include <cfloat>

namespace gmm {

constexpr int kModeTile = 32;            // points per CTA
constexpr int kModeThreads = 128;        // a quad of 4 threads per point
constexpr int kModeChunk = 8;            // component records per shared-memory chunk
constexpr int kModeRound = 16;           // iterations per round of mode_iter_kernel
constexpr int kModeScanThreads = 1024;   // candidates per block of the compaction
constexpr int kModeLabelThreads = 128;   // points per block of mode_label_kernel
enum { kModeActive = 0, kModeConverged = 1, kModeUnconverged = 2, kModeNotFinite = 3 };

__host__ __device__ constexpr int mode_np(int DP) { return DP * (DP + 1) / 2; }
__host__ __device__ constexpr int mode_rec_floats(int DP) { return DP + DP * DP + 4; }
__host__ __device__ constexpr int mode_apitch(int DP) { return mode_np(DP) | 1; }          // odd: no bank conflicts
// dynamic shared memory of mode_iter_kernel<DP>: records, weights, A, delta / g, per-point scalars, then the (i, j) table
__host__ __device__ constexpr size_t mode_iter_smem(int DP) {
    return sizeof(float) * ((size_t)kModeChunk * mode_rec_floats(DP) + kModeTile * kModeChunk + (size_t)kModeTile * mode_apitch(DP) +
                            2 * kModeTile * DP + 4 * kModeTile) + sizeof(int) * mode_np(DP);
}

// The start of every point: x = src[e * row_stride + d * dim_stride] - shift[d] (shift NULL: no shift) for d < D, 0 beyond,
// into xs [n][DP]; iters = 0; status kModeActive, or kModeNotFinite when a coordinate is not finite.
__global__ void __launch_bounds__(256)
mode_init_kernel(const float* __restrict__ src, long long row_stride, long long dim_stride, int n, int D, int DP,
                 const float* __restrict__ shift, float* __restrict__ xs, int* __restrict__ iters, int* __restrict__ status) {
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= n) return;
    bool finite = true;
    for (int d = 0; d < DP; d++) {
        float v = 0.0f;
        if (d < D) {
            v = src[(long long)e * row_stride + (long long)d * dim_stride];
            finite = finite && isfinite(v);
            if (shift) v = __fsub_rn(v, shift[d]);
        }
        xs[(size_t)e * DP + d] = v;
    }
    iters[e] = 0;
    status[e] = finite ? kModeActive : kModeNotFinite;
}

// Order-preserving compaction of the active points, without atomics.  Candidates are idx[0 .. m) (idx NULL: 0 .. m); pass 1
// counts the active ones per block of kModeScanThreads into bcount, pass 2 scans the block counts (one block; the total to
// *count), pass 3 writes each active candidate to out[block offset + its rank in the block].
__device__ __forceinline__ int mode_block_rank(bool flag, int* warp_tot, int* total) {
    const unsigned ball = __ballot_sync(0xffffffffu, flag);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_tot[w] = __popc(ball);
    __syncthreads();
    if (w == 0) {
        const int v = warp_tot[lane];
        int s = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        warp_tot[lane] = s - v;                           // exclusive prefix of the warps
        if (lane == 31) *total = s;
    }
    __syncthreads();
    return warp_tot[w] + __popc(ball & ((1u << lane) - 1u));
}
__global__ void __launch_bounds__(kModeScanThreads)
mode_count_kernel(const int* __restrict__ idx, int m, const int* __restrict__ status, int* __restrict__ bcount) {
    __shared__ int wt[32], tot;
    const int i = blockIdx.x * kModeScanThreads + threadIdx.x;
    const bool f = i < m && status[idx ? idx[i] : i] == kModeActive;
    mode_block_rank(f, wt, &tot);
    if (threadIdx.x == 0) bcount[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(kModeScanThreads)
mode_scan_kernel(int* __restrict__ bcount, int nb, int* __restrict__ count) {
    __shared__ int wt[32], tot;
    int base = 0;
    for (int b0 = 0; b0 < nb; b0 += kModeScanThreads) {
        const int b = b0 + threadIdx.x;
        const int v = b < nb ? bcount[b] : 0;
        // ranks of unit flags would not do: a block count is up to 1024.  Inclusive scan of v in the block, in fixed order
        int s = v;
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        if (lane == 31) wt[w] = s;
        __syncthreads();
        if (w == 0) {
            const int x = wt[lane];
            int y = x;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, y, o);
                if (lane >= o) y += t;
            }
            wt[lane] = y - x;
            if (lane == 31) tot = y;
        }
        __syncthreads();
        if (b < nb) bcount[b] = base + wt[w] + s - v;    // exclusive offset of block b
        base += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = base;
}
__global__ void __launch_bounds__(kModeScanThreads)
mode_scatter_kernel(const int* __restrict__ idx, int m, const int* __restrict__ status, const int* __restrict__ boff,
                    int* __restrict__ out) {
    __shared__ int wt[32], tot;
    const int i = blockIdx.x * kModeScanThreads + threadIdx.x;
    const int e = i < m ? (idx ? idx[i] : i) : 0;
    const bool f = i < m && status[e] == kModeActive;
    const int r = mode_block_rank(f, wt, &tot);
    if (f) out[boff[blockIdx.x] + r] = e;
}

// Up to `round` iterations of the points active[0 .. na), each stopping on its own (status, iters and xs updated in place).
// A CTA holds kModeTile points; the quad of point q (threads 4q .. 4q + 3) keeps x in registers and owns the rows
// [lane * DP / 4, (lane + 1) * DP / 4) of v = S_k dx_k and g.  Per chunk of kModeChunk records:
//   logits  each quad, component by component in increasing k: v's rows, q = dx^T v (the four row sums added
//           pairwise: (q0 + q1) + (q2 + q3) on every lane), l = const - q / 2, the online log-sum-exp (m, s) and
//           g = g exp(m_old - m_new) - w v with w = exp(l - m_new), exactly as condition_simt_kernel rescales its moments;
//   A       after the chunk: A = A exp(m_start - m_end) + sum_kk exp(l_kk - m_end) S_kk, each packed entry (i >= j) of
//           each point a fixed fma chain in increasing kk, over a register tile of 8 points per thread.
// Then one thread per point factors its A (padded diagonal set to 1) in shared memory, solves A delta = g, and
// decides: a pivot that is not positive or a delta that is not finite -> kModeUnconverged (x kept); else x += delta and,
// when max_d |delta_d| inv_sigma_d < tol, kModeConverged, or when iters reaches max_iter, kModeUnconverged.
// g and A carry the same factor exp(-m) and it cancels in delta.  A point's arithmetic depends only on its own x and the
// records, never on its CTA, slot or round.
template <int DP>
__global__ void __launch_bounds__(kModeThreads, 1)
mode_iter_kernel(int D, int Kp, const float* __restrict__ rec, const float* __restrict__ inv_sigma, const int* __restrict__ active,
                 int na, float* __restrict__ xs, int* __restrict__ iters, int* __restrict__ status, int max_iter, float tol, int round) {
    constexpr int REC = mode_rec_floats(DP), NP = mode_np(DP), AP = mode_apitch(DP), RW = DP / 4, KC = kModeChunk, T = kModeTile;
    extern __shared__ __align__(16) float smem[];
    float* srec = smem;                                  // [KC][REC]
    float* sW = srec + KC * REC;                         // [T][KC] weights of the chunk
    float* sA = sW + T * KC;                             // [T][AP] packed lower triangle of A, then its Cholesky factor
    float* sD = sA + T * AP;                             // [T][DP] g, then delta
    float* sX = sD + T * DP;                             // [T][DP] x before the step
    float* sScale = sX + T * DP;                         // [T] exp(m_start - m_end) of the chunk
    int* sState = reinterpret_cast<int*>(sScale + T);    // [T] status after the step
    int* sMove = sState + T;                             // [T] 1: x += delta
    int* sPair = sMove + 2 * T;                          // [NP] (i << 8) | j of packed entry c

    for (int c = threadIdx.x; c < NP; c += kModeThreads) {
        int i = 0;
        while ((i + 1) * (i + 2) / 2 <= c) i++;
        sPair[c] = (i << 8) | (c - i * (i + 1) / 2);
    }
    const int q = threadIdx.x >> 2, lane = threadIdx.x & 3, r0 = lane * RW;
    const int slot = blockIdx.x * T + q;
    const bool valid = slot < na;
    const int e = valid ? active[slot] : 0;
    float x[DP], xr[RW];
#pragma unroll
    for (int d = 0; d < DP; d++) x[d] = valid ? xs[(size_t)e * DP + d] : 0.0f;
#pragma unroll
    for (int i = 0; i < RW; i++) xr[i] = valid ? xs[(size_t)e * DP + r0 + i] : 0.0f;
    int it = valid ? iters[e] : 0, st = valid ? status[e] : kModeConverged;

    for (int r = 0; r < round; r++) {
        const bool act = st == kModeActive && it < max_iter;
        if (!__syncthreads_or(act)) break;
        float m = -FLT_MAX, s = 0.0f, g[RW];
#pragma unroll
        for (int i = 0; i < RW; i++) g[i] = 0.0f;
        for (int k0 = 0; k0 < Kp; k0 += KC) {
            __syncthreads();
            {
                const float4* src = reinterpret_cast<const float4*>(rec + (size_t)k0 * REC);
                float4* dst = reinterpret_cast<float4*>(srec);
                for (int i = threadIdx.x; i < KC * REC / 4; i += kModeThreads) dst[i] = src[i];
            }
            __syncthreads();
            const float m_start = m;
#pragma unroll
            for (int kk = 0; kk < KC; kk++) {
                const float* p = srec + kk * REC;
                float dx[DP];
#pragma unroll
                for (int d = 0; d < DP; d++) dx[d] = x[d] - p[d];
                float v[RW], qp = 0.0f;
#pragma unroll
                for (int i = 0; i < RW; i++) {
                    const float* row = p + DP + (r0 + i) * DP;
                    float t = 0.0f;
#pragma unroll
                    for (int j = 0; j < DP; j++) t = fmaf(row[j], dx[j], t);
                    v[i] = t;
                    qp = fmaf(xr[i] - p[r0 + i], t, qp);
                }
                float qs = qp + __shfl_xor_sync(0xffffffffu, qp, 1);
                qs = qs + __shfl_xor_sync(0xffffffffu, qs, 2);
                const float l = fmaf(-0.5f, qs, p[DP + DP * DP]);
                const float m2 = fmaxf(m, l);
                const float rs = expf(m - m2), w = expf(l - m2);
                s = fmaf(s, rs, w);
#pragma unroll
                for (int i = 0; i < RW; i++) g[i] = fmaf(-w, v[i], __fmul_rn(g[i], rs));
                m = m2;
                if (lane == 0) sW[q * KC + kk] = l;
            }
            if (lane == 0) {
#pragma unroll
                for (int kk = 0; kk < KC; kk++) sW[q * KC + kk] = expf(sW[q * KC + kk] - m);
                sScale[q] = expf(m_start - m);
            }
            __syncthreads();
            for (int item = threadIdx.x; item < NP * (T / 8); item += kModeThreads) {
                const int c = item % NP, e0 = (item / NP) * 8;
                const int ij = sPair[c];
                const float* sc = srec + DP + (ij >> 8) * DP + (ij & 255);
                float sv[KC];
#pragma unroll
                for (int kk = 0; kk < KC; kk++) sv[kk] = sc[kk * REC];
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    float* a = sA + (e0 + t) * AP + c;
                    float acc = k0 == 0 ? 0.0f : __fmul_rn(*a, sScale[e0 + t]);
#pragma unroll
                    for (int kk = 0; kk < KC; kk++) acc = fmaf(sW[(e0 + t) * KC + kk], sv[kk], acc);
                    *a = acc;
                }
            }
        }
#pragma unroll
        for (int i = 0; i < RW; i++) { sD[q * DP + r0 + i] = g[i]; sX[q * DP + r0 + i] = xr[i]; }
        __syncthreads();
        if (threadIdx.x < T) {
            const int p = threadIdx.x;
            float* A = sA + p * AP;
            float* b = sD + p * DP;
            for (int d = D; d < DP; d++) A[d * (d + 1) / 2 + d] = 1.0f;
            bool ok = true;
            for (int j = 0; j < DP && ok; j++) {
                float* Lj = A + j * (j + 1) / 2;
                float t = Lj[j];
                for (int k = 0; k < j; k++) t = fmaf(-Lj[k], Lj[k], t);
                if (!(t > 0.0f)) { ok = false; break; }
                const float inv = rsqrtf(t);                        // the factor's diagonal is kept as its reciprocal
                Lj[j] = inv;
                for (int i = j + 1; i < DP; i++) {
                    float* Li = A + i * (i + 1) / 2;
                    float u = Li[j];
                    for (int k = 0; k < j; k++) u = fmaf(-Li[k], Lj[k], u);
                    Li[j] = u * inv;
                }
            }
            bool small = true;
            if (ok) {
                for (int i = 0; i < DP; i++) {                       // L y = g
                    const float* Li = A + i * (i + 1) / 2;
                    float u = b[i];
                    for (int k = 0; k < i; k++) u = fmaf(-Li[k], b[k], u);
                    b[i] = u * Li[i];
                }
                for (int i = DP - 1; i >= 0; i--) {                  // L^T delta = y
                    float u = b[i];
                    for (int k = i + 1; k < DP; k++) u = fmaf(-A[k * (k + 1) / 2 + i], b[k], u);
                    b[i] = u * A[i * (i + 1) / 2 + i];
                    ok = ok && isfinite(b[i]);
                    // below tol sigma_d, or within 2 ulp of x_d: farther than about tol / 2^-22 spreads from the centre a
                    // float coordinate cannot resolve tol sigma_d, and the step would only hop between neighbours
                    small = small && fabsf(b[i]) * inv_sigma[i] < fmaxf(tol, fabsf(sX[p * DP + i]) * 0x1p-22f * inv_sigma[i]);
                }
            }
            sMove[p] = ok;
            sState[p] = !ok ? kModeUnconverged : small ? kModeConverged : kModeActive;
        }
        __syncthreads();
        if (act) {
            if (sMove[q]) {
#pragma unroll
                for (int d = 0; d < DP; d++) x[d] = x[d] + sD[q * DP + d];
#pragma unroll
                for (int i = 0; i < RW; i++) xr[i] = xr[i] + sD[q * DP + r0 + i];
            }
            it++;
            st = sState[q];
            if (st == kModeActive && it >= max_iter) st = kModeUnconverged;
        }
    }
    if (valid) {
#pragma unroll
        for (int i = 0; i < RW; i++) xs[(size_t)e * DP + r0 + i] = xr[i];
        if (lane == 0) { iters[e] = it; status[e] = st; }
    }
}

// The outcome of every point, one thread per point: logp = ln p at the endpoint (the records streamed through shared
// memory in chunks; per record one fma chain over the full rows of S dx, so not bit-equal to the iteration's quad-split
// logits, then an online log-sum-exp); the label
// (kModeConverged: the mode of smallest rho = max_d |x_d - mode_d| inv_sigma_d with rho <= merge_tol, ties to the lower
// index, -2 when none; otherwise -1); the endpoint x + shift in absolute float coordinates (NaN for kModeNotFinite).
// modes: [n_modes][DP] relative to the centre.  endpoints [n][D] and logp may be NULL.
template <int DP>
__global__ void __launch_bounds__(kModeLabelThreads, 1)
mode_label_kernel(int n, int D, int Kp, const float* __restrict__ rec, const float* __restrict__ inv_sigma,
                  const float* __restrict__ modes, int n_modes, float merge_tol, const float* __restrict__ xs,
                  const int* __restrict__ status, const float* __restrict__ shift, int* __restrict__ labels,
                  float* __restrict__ endpoints, float* __restrict__ logp) {
    constexpr int REC = mode_rec_floats(DP), KC = kModeChunk;
    __shared__ __align__(16) float srec[KC * REC];
    const int e = blockIdx.x * kModeLabelThreads + threadIdx.x;
    const bool valid = e < n;
    float x[DP];
#pragma unroll
    for (int d = 0; d < DP; d++) x[d] = valid ? xs[(size_t)e * DP + d] : 0.0f;
    const int st = valid ? status[e] : kModeNotFinite;
    float m = -FLT_MAX, s = 0.0f;
    if (logp) {
        for (int k0 = 0; k0 < Kp; k0 += KC) {
            __syncthreads();
            {
                const float4* src = reinterpret_cast<const float4*>(rec + (size_t)k0 * REC);
                float4* dst = reinterpret_cast<float4*>(srec);
                for (int i = threadIdx.x; i < KC * REC / 4; i += kModeLabelThreads) dst[i] = src[i];
            }
            __syncthreads();
            for (int kk = 0; kk < KC; kk++) {
                const float* p = srec + kk * REC;
                float dx[DP];
#pragma unroll
                for (int d = 0; d < DP; d++) dx[d] = x[d] - p[d];
                float qs = 0.0f;
#pragma unroll
                for (int i = 0; i < DP; i++) {
                    float t = 0.0f;
#pragma unroll
                    for (int j = 0; j < DP; j++) t = fmaf(p[DP + i * DP + j], dx[j], t);
                    qs = fmaf(dx[i], t, qs);
                }
                const float l = fmaf(-0.5f, qs, p[DP + DP * DP]);
                const float m2 = fmaxf(m, l);
                s = fmaf(s, expf(m - m2), expf(l - m2));
                m = m2;
            }
        }
    }
    if (!valid) return;
    int lab = -1;
    if (st == kModeConverged) {
        float best = INFINITY;
        lab = -2;
        for (int j = 0; j < n_modes; j++) {
            float rho = 0.0f;
#pragma unroll
            for (int d = 0; d < DP; d++) rho = fmaxf(rho, fabsf(x[d] - modes[(size_t)j * DP + d]) * inv_sigma[d]);
            if (rho <= merge_tol && rho < best) { best = rho; lab = j; }
        }
    }
    labels[e] = lab;
    const float nan = __int_as_float(0x7fc00000);
    if (endpoints) {
#pragma unroll
        for (int d = 0; d < DP; d++)
            if (d < D) endpoints[(size_t)e * D + d] = st == kModeNotFinite ? nan : __fadd_rn(x[d], shift[d]);
    }
    if (logp) logp[e] = st == kModeNotFinite ? nan : m + logf(s);
}

}  // namespace gmm
