// kernels_simt.cuh — CUDA-core (SIMT) kernels of the EM hot path for sm_90a.
//
// These are the reference-arithmetic GPU kernels: FP32 quadratic form exactly
// as estep1 forms it ((x - mu) first, then the D x D form), FP64 accumulation
// of the M-step statistics.  They are the accuracy anchor on the device and the
// path for shapes the wgmma kernels do not cover.  Layouts:
//   xs    : events SoA  [D][xpitch] (device transpose of the AoS shard, rows pitched to 32 events; the
//           reference keeps the same copy: gaussian.cu:209-218, 373-377)
//   memb  : responsibilities, cluster-major [K][n] (gaussian.h:75)
//   stats : per cluster F = 1 + D + D(D+1)/2 doubles
//           [ sum g | sum g (x-s)_d | sum g (x-s)_i (x-s)_j, i>=j ] then 1 LL slot
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace gmm {

__host__ __device__ constexpr int epack_stride_c(int D) {
    return ((((D + 3) & ~3) + D * (D + 1) / 2 + 1) + 3) & ~3;
}
constexpr int kEstepClusterChunk = 16;
constexpr int kEstepThreads = 128;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------
// E-step: estep1 + estep2 of the reference (gaussian_kernel.cu:383-512) fused
// in one pass.  One thread per event, event held in registers, the cluster
// parameters (mean, combined symmetric coefficients, constant + ln pi) staged
// through shared memory in chunks of 16 clusters.  Unnormalised log numerators
// go to memb while a running max / sum-exp is kept (online log-sum-exp); the
// second sweep re-reads them (L2-resident: the block wrote them microseconds
// ago) and stores exp(l - denom).  The per-event log-likelihood terms are
// reduced in double and added to *ll_out.
// ---------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kEstepThreads)
estep_simt_kernel(const float* __restrict__ xs, size_t xpitch, int n, int K, const float* __restrict__ epack,
                  float* __restrict__ memb, size_t pitch, double* __restrict__ ll_out) {
    constexpr int STRIDE = epack_stride_c(D);
    constexpr int COEF = (D + 3) & ~3;
    constexpr int NCOEF = D * (D + 1) / 2;
    __shared__ __align__(16) float sp[kEstepClusterChunk * STRIDE];
    __shared__ double sred[kEstepThreads / 32];

    const int e = blockIdx.x * kEstepThreads + threadIdx.x;
    const bool valid = e < n;
    float x[D];
#pragma unroll
    for (int d = 0; d < D; d++) x[d] = valid ? xs[(size_t)d * xpitch + e] : 0.0f;

    float run_max = -INFINITY, run_sum = 0.0f;
    for (int k0 = 0; k0 < K; k0 += kEstepClusterChunk) {
        const int kc = min(kEstepClusterChunk, K - k0);
        __syncthreads();
        {
            const float4* src = reinterpret_cast<const float4*>(epack + (size_t)k0 * STRIDE);
            float4* dst = reinterpret_cast<float4*>(sp);
            for (int i = threadIdx.x; i < kc * STRIDE / 4; i += kEstepThreads) dst[i] = src[i];
        }
        __syncthreads();
        for (int kk = 0; kk < kc; kk++) {
            const float* p = sp + kk * STRIDE;
            float dx[D];
#pragma unroll
            for (int d = 0; d < D; d++) dx[d] = x[d] - p[d];
            float q = 0.0f;
            int idx = COEF;
#pragma unroll
            for (int i = 0; i < D; i++) {
                float t = 0.0f;
#pragma unroll
                for (int j = i; j < D; j++) t = fmaf(p[idx++], dx[j], t);
                q = fmaf(dx[i], t, q);
            }
            const float l = fmaf(-0.5f, q, p[COEF + NCOEF]);
            if (valid) memb[(size_t)(k0 + kk) * pitch + e] = l;
            const float m2 = fmaxf(run_max, l);
            run_sum = run_sum * expf(run_max - m2) + expf(l - m2);
            run_max = m2;
        }
    }
    const float denom = run_max + logf(run_sum);            // estep2 :490-494
    if (valid) {
        for (int k = 0; k < K; k++) {
            float* g = memb + (size_t)k * pitch + e;
            *g = expf(*g - denom);                          // estep2 :498-501
        }
    }
    double ll = valid ? (double)denom : 0.0;
    ll = warp_sum(ll);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = ll;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
#pragma unroll
        for (int w = 0; w < kEstepThreads / 32; w++) s += sred[w];
        atomicAdd(ll_out, s);
    }
}

// ---------------------------------------------------------------------------
// M-step statistics: mstep_N + mstep_means + mstep_covariance1 of the
// reference (gaussian_kernel.cu:522-677) as ONE pass over the events and the
// responsibilities:  stats[k][f] += sum_n g[k][n] * phi_f(x_n - shift), with
// phi = [1, x, x_i x_j (i>=j)].  This is a (K x n) . (n x F) product; here it
// runs on the FP64 CUDA cores (products of two floats are exact in double, so
// the statistics are exact up to the final double rounding) — it is the
// accuracy anchor for the wgmma path, not the fast path.
// Thread layout: 256 threads = 16 (cluster groups of CPT) x 16 (feature lanes,
// JMAX features each); TE events per shared-memory tile.
// ---------------------------------------------------------------------------
constexpr int kMstepThreads = 256;
constexpr int kMstepTE = 32;

template <int JMAX, int CPT>
__global__ void __launch_bounds__(kMstepThreads, 1)
mstep_simt_kernel(const float* __restrict__ xs, size_t xpitch, int n, int D, int K, const float* __restrict__ memb, size_t pitch,
                  const double* __restrict__ shift, double* __restrict__ stats, int events_per_block) {
    constexpr int FP = 16 * JMAX;          // padded feature count
    constexpr int KT = 16 * CPT;           // clusters per block
    constexpr int GS = KT + 2;             // padded row of the gamma tile (16-byte aligned rows)
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* phi = reinterpret_cast<double*>(smem_raw);            // [TE][FP]
    double* gt = phi + kMstepTE * FP;                             // [TE][GS]
    double* xt = gt + kMstepTE * GS;                              // [TE][D]
    short* fi = reinterpret_cast<short*>(xt + kMstepTE * GMM_MAX_DIMENSIONS);   // [FP]
    short* fj = fi + FP;

    const int F = 1 + D + D * (D + 1) / 2;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int k0 = blockIdx.y * KT;

    for (int f = tid; f < FP; f += kMstepThreads) {               // feature -> (i, j) table
        short a = -1, b = -1;                                     // -1: constant one / zero pad
        if (f >= 1 && f <= D) { a = (short)(f - 1); b = -2; }     // linear feature
        else if (f > D && f < F) {
            int t = f - 1 - D, i = 0;
            while ((i + 1) * (i + 2) / 2 <= t) i++;
            a = (short)i; b = (short)(t - i * (i + 1) / 2);
        } else if (f >= F) { a = -3; }
        fi[f] = a; fj[f] = b;
    }

    double acc[CPT][JMAX];
#pragma unroll
    for (int c = 0; c < CPT; c++)
#pragma unroll
        for (int j = 0; j < JMAX; j++) acc[c][j] = 0.0;

    const long long ebeg = (long long)blockIdx.x * events_per_block;
    const long long eend = min((long long)n, ebeg + events_per_block);

    for (long long e0 = ebeg; e0 < eend; e0 += kMstepTE) {
        __syncthreads();
        for (int idx = tid; idx < kMstepTE * D; idx += kMstepThreads) {       // shifted events
            const int d = idx / kMstepTE, t = idx % kMstepTE;
            const long long e = e0 + t;
            xt[t * GMM_MAX_DIMENSIONS + d] = (e < eend) ? (double)xs[(size_t)d * xpitch + e] - shift[d] : 0.0;
        }
        for (int idx = tid; idx < kMstepTE * KT; idx += kMstepThreads) {      // responsibilities
            const int kk = idx / kMstepTE, t = idx % kMstepTE;
            const long long e = e0 + t;
            const int k = k0 + kk;
            gt[t * GS + kk] = (k < K && e < eend) ? (double)memb[(size_t)k * pitch + e] : 0.0;
        }
        __syncthreads();
        for (int idx = tid; idx < kMstepTE * FP; idx += kMstepThreads) {      // features
            const int t = idx / FP, f = idx % FP;
            const short a = fi[f], b = fj[f];
            double v;
            if (a == -1) v = 1.0;
            else if (a == -3) v = 0.0;
            else if (b == -2) v = xt[t * GMM_MAX_DIMENSIONS + a];
            else v = xt[t * GMM_MAX_DIMENSIONS + a] * xt[t * GMM_MAX_DIMENSIONS + b];
            phi[t * FP + f] = v;
        }
        __syncthreads();
#pragma unroll 2
        for (int t = 0; t < kMstepTE; t++) {
            double g[CPT];
#pragma unroll
            for (int c = 0; c < CPT; c++) g[c] = gt[t * GS + ty * CPT + c];
#pragma unroll
            for (int j = 0; j < JMAX; j++) {
                const double p = phi[t * FP + tx + 16 * j];
#pragma unroll
                for (int c = 0; c < CPT; c++) acc[c][j] = fma(g[c], p, acc[c][j]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < CPT; c++) {
        const int k = k0 + ty * CPT + c;
        if (k < K) {
#pragma unroll
            for (int j = 0; j < JMAX; j++) {
                const int f = tx + 16 * j;
                if (f < F) atomicAdd(&stats[(size_t)k * F + f], acc[c][j]);
            }
        }
    }
}

// AoS [n][D] -> SoA [D][n] (gaussian.cu:212-218 done on the device).
__global__ void transpose_aos_to_soa_kernel(const float* __restrict__ aos, float* __restrict__ soa, size_t xpitch, int n, int D) {
    __shared__ float tile[32][33];
    const int e0 = blockIdx.x * 32;
    for (int d0 = 0; d0 < D; d0 += 32) {
        // read: 32 events x 32 dims, contiguous along d within an event
        for (int r = threadIdx.y; r < 32; r += blockDim.y) {
            const int e = e0 + r, d = d0 + threadIdx.x;
            tile[r][threadIdx.x] = (e < n && d < D) ? aos[(size_t)e * D + d] : 0.0f;
        }
        __syncthreads();
        for (int r = threadIdx.y; r < 32; r += blockDim.y) {
            const int d = d0 + r, e = e0 + threadIdx.x;
            if (d < D && e < n) soa[(size_t)d * xpitch + e] = tile[threadIdx.x][r];
        }
        __syncthreads();
    }
}

// Column sums for seeding: out[d] += sum x, out[D+d] += sum x^2 (double); column extremes:
// out[2D+d] = max x, out[3D+d] = max (-x) (initialised to -DBL_MAX by the caller).
// Replaces mvtmeans / averageVariance (gaussian_kernel.cu:54-102), which scan
// the events serially with one thread per dimension.
__device__ __forceinline__ void atomic_max_double(double* addr, double v) {
    unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
    unsigned long long old = *a;
    while (__longlong_as_double((long long)old) < v) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
}
__global__ void column_moments_kernel(const float* __restrict__ xs, size_t xpitch, int n, int D, double* __restrict__ out) {
    const int d = blockIdx.y;
    const float* col = xs + (size_t)d * xpitch;
    double s1 = 0, s2 = 0;
    float mx = -INFINITY, mn = INFINITY;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const float x = col[e];
        const double v = x;
        s1 += v;
        s2 += v * v;
        mx = fmaxf(mx, x);
        mn = fminf(mn, x);
    }
    __shared__ double r1[8], r2[8];
    __shared__ float r3[8], r4[8];
    s1 = warp_sum(s1); s2 = warp_sum(s2);
    for (int o = 16; o > 0; o >>= 1) { mx = fmaxf(mx, __shfl_down_sync(0xffffffffu, mx, o)); mn = fminf(mn, __shfl_down_sync(0xffffffffu, mn, o)); }
    if ((threadIdx.x & 31) == 0) { r1[threadIdx.x >> 5] = s1; r2[threadIdx.x >> 5] = s2; r3[threadIdx.x >> 5] = mx; r4[threadIdx.x >> 5] = mn; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0;
        float hi = -INFINITY, lo = INFINITY;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) { a += r1[w]; b += r2[w]; hi = fmaxf(hi, r3[w]); lo = fminf(lo, r4[w]); }
        atomicAdd(&out[d], a);
        atomicAdd(&out[D + d], b);
        if (hi >= lo) {                                      // this block saw at least one event
            atomic_max_double(&out[2 * D + d], (double)hi);
            atomic_max_double(&out[3 * D + d], -(double)lo);
        }
    }
}

}  // namespace gmm
