// kernels_condition.cuh — gmm_condition's imputing kernel, for sm_90a.
//
// Events measured on the observed dimensions O only are scored under the marginal mixture sum_k pi_k N(x_O | mu_kO, R_kOO)
// and the missing dimensions M get the moments of the conditional mixture (the semantics are spelt out in gmm.h):
//   m_k = mu_kM + G_k dx,  dx = x_O - mu_kO,  G_k = -P_kMM^-1 P_kMO      (conditional mean of component k)
//   c_k = diag(P_kMM^-1)                                                (conditional variance of component k)
//   E[x_M | x_O] = sum_k r_k m_k,  Var[x_M | x_O]_dd = sum_k r_k (c_kd + (m_kd - E_d)^2),  r_k the posterior.
// The host derives the per-cluster parameters in double and rounds them to float.  Parameter block: one record of
// cond_rec_floats(NO, NM) floats per cluster, NO and NM the observed / imputed counts rounded up to a multiple of 4:
//   [ epack record of the NO-dimensional marginal (mu_O | coefficients of P_O | constant_O + ln pi) | mu_M (NM) |
//     G row-major (NM x NO) | c (NM) ], zero beyond the real counts.
#pragma once
#include <cuda_runtime.h>
#include "kernels_simt.cuh"

namespace gmm {

__host__ __device__ constexpr int cond_round4(int v) { return (v + 3) & ~3; }
__host__ __device__ constexpr int cond_rec_floats(int NO, int NM) { return epack_stride_c(NO) + NM * (NO + 2); }

// One thread per event.  Per cluster: GMM_SCORE_CLUSTER's logit (the marginal), then m_k from the same dx, merged into a
// running weight W = run_sum, mean and M2 = sum_k w_k (c_k + (m_k - mean)^2) by the weighted update of West (1979):
// with the earlier weight W0 scaled to the new maximum by `rescale`, W' = W0 + w, delta = m_k - mean,
//   mean += delta w / W',  M2 = M2 rescale + w (c_k + delta^2 W0 / W').
// No term is a difference of large numbers, so the variance keeps its precision on raw intensities of 1e4 and more.
// cond_mean / cond_var: [n][n_mis] (cond_var may be NULL); labels, max_resp, logp and *ll_out as score_simt_kernel.
// The minimum of one block per SM lets ptxas use the registers it needs (at most 150): without it, it spilled a few words
// in a third of the instances at under 140 registers.
template <int NO, int NM>
__global__ void __launch_bounds__(kEstepThreads, 1)
condition_simt_kernel(const float* __restrict__ x_obs, int n, int n_obs, int n_mis, int K, const float* __restrict__ cpack,
                      int* __restrict__ labels, float* __restrict__ max_resp, float* __restrict__ logp, double* __restrict__ ll_out,
                      float* __restrict__ cond_mean, float* __restrict__ cond_var) {
    constexpr int STRIDE = cond_rec_floats(NO, NM);
    constexpr int EP = epack_stride_c(NO);
    __shared__ __align__(16) float sp[kEstepClusterChunk * STRIDE];
    __shared__ double sred[kEstepThreads / 32];

    const int e = blockIdx.x * kEstepThreads + threadIdx.x;
    const bool valid = e < n;
    float x[NO];
#pragma unroll
    for (int d = 0; d < NO; d++) x[d] = (valid && d < n_obs) ? x_obs[(size_t)e * n_obs + d] : 0.0f;

    float run_max = -FLT_MAX, run_sum = 0.0f, best_l = -INFINITY;        // -FLT_MAX: pi = 0 adds 0 (estep_simt_kernel)
    int best_k = -1;
    float mean[NM], m2[NM];
#pragma unroll
    for (int d = 0; d < NM; d++) { mean[d] = 0.0f; m2[d] = 0.0f; }
    for (int k0 = 0; k0 < K; k0 += kEstepClusterChunk) {
        const int kc = min(kEstepClusterChunk, K - k0);
        __syncthreads();
        {
            const float4* src = reinterpret_cast<const float4*>(cpack + (size_t)k0 * STRIDE);
            float4* dst = reinterpret_cast<float4*>(sp);
            for (int i = threadIdx.x; i < kc * STRIDE / 4; i += kEstepThreads) dst[i] = src[i];
        }
        __syncthreads();
        for (int kk = 0; kk < kc; kk++) {
            const float* p = sp + kk * STRIDE;
            const float max0 = run_max, sum0 = run_sum;
            GMM_SCORE_CLUSTER(NO, x, p, k0 + kk, dx, l, run_max, run_sum, best_l, best_k)
            const float rescale = expf(max0 - run_max);    // the factors the log-sum-exp just applied
            const float w = expf(l - run_max);
            // the earlier weight at the new maximum.  __fmul_rn: a plain product would be shared with the log-sum-exp's
            // run_sum * rescale + w, which then is no longer contracted to one fma and differs from score_simt_kernel's
            const float w0 = __fmul_rn(sum0, rescale);
            // run_sum is in [1, K] (the maximum's own term is 1): the fast division is safe and its 2 ulp are harmless here;
            // the IEEE division's slow-path call would make ptxas spill around it (also below).  It is 0 while every logit so
            // far is -inf (pi = 0): the floor at FLT_MIN then makes f = g = 0 (not 0 / 0) and leaves mean and M2 at 0
            const float rs = fmaxf(run_sum, FLT_MIN);
            const float f = __fdividef(w, rs), g = __fdividef(w0, rs);
            const float* mu = p + EP;
            const float* G = mu + NM;
            const float* cv = G + NM * NO;
#pragma unroll
            for (int d = 0; d < NM; d++) {
                float t = 0.0f;
#pragma unroll
                for (int j = 0; j < NO; j++) t = fmaf(G[d * NO + j], dx[j], t);
                const float delta = (mu[d] + t) - mean[d];
                mean[d] = fmaf(delta, f, mean[d]);
                m2[d] = fmaf(m2[d], rescale, w * fmaf(delta * delta, g, cv[d]));
            }
        }
    }
    if (valid) {
        float* om = cond_mean + (size_t)e * n_mis;
#pragma unroll
        for (int d = 0; d < NM; d++)
            if (d < n_mis) om[d] = mean[d];
        if (cond_var) {
            float* ov = cond_var + (size_t)e * n_mis;
#pragma unroll
            for (int d = 0; d < NM; d++)
                if (d < n_mis) ov[d] = __fdividef(m2[d], run_sum);
        }
    }
    const float denom = run_max + logf(run_sum);         // score_simt_kernel's end
    if (valid) {
        labels[e] = best_k;
        max_resp[e] = best_k >= 0 ? expf(best_l - denom) : __int_as_float(0x7fc00000);
        logp[e] = denom;
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

// Chunk preparation of gmm_condition_stats: ONE pass over a chunk's rows [n][n_obs] (the coordinates of the observed
// dimensions) that writes
//   xo_soa[a][e] = x                the observed SoA copy [n_obs][pitch] the marginal E-step reads (when xo_soa != NULL);
//   the D-row image [D][pitch] the context's M-step reads, so that the missing dimensions add exact zeros (when
//   shift_f is the float centre the M-step uses) and the observed entries of its output are the marginal moments:
//     z_img (wgmma M-step)  (x - shift_f) * inv_scale_f on an observed row, with standardise_soa_kernel's operations
//                           (bit-identical to score_stats_prep_kernel's z), and 0 on a missing row;
//     x_img (FP64 M-step)   x on an observed row and shift_f on a missing row;
//   *flag |= kScoreStatsNotFinite for a coordinate that is not finite, kScoreStatsBeyondZb for |z| >= zb on an observed
//            dimension (tested when z_img != NULL).
// obs_mask: bit d set when dimension d is observed (its column in the rows is the number of observed dimensions below it).
// Block (32, 8), as score_stats_prep_kernel.
__global__ void __launch_bounds__(256)
condition_stats_prep_kernel(const float* __restrict__ rows_obs, int n, int n_obs, int D, unsigned obs_mask,
                            const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f, float zb,
                            float* __restrict__ xo_soa, float* __restrict__ z_img, float* __restrict__ x_img, size_t pitch,
                            int* __restrict__ flag) {
    __shared__ float tile[32][33];
    const int e0 = blockIdx.x * 32;
    const int rows = min(32, n - e0);
    const int tid = threadIdx.y * 32 + threadIdx.x;
    const float* src = rows_obs + (size_t)e0 * n_obs;
    for (int i = tid; i < rows * n_obs; i += 256) tile[i / n_obs][i % n_obs] = src[i];
    __syncthreads();
    const int e = e0 + threadIdx.x;
    int bits = 0;
    if (threadIdx.x < rows) {
        for (int d = threadIdx.y; d < D; d += 8) {
            if (!((obs_mask >> d) & 1u)) {
                if (z_img) z_img[(size_t)d * pitch + e] = 0.0f;
                if (x_img) x_img[(size_t)d * pitch + e] = shift_f[d];
                continue;
            }
            const int a = __popc(obs_mask & ((1u << d) - 1u));
            const float x = tile[threadIdx.x][a];
            if (!isfinite(x)) bits |= kScoreStatsNotFinite;
            if (xo_soa) xo_soa[(size_t)a * pitch + e] = x;
            if (x_img) x_img[(size_t)d * pitch + e] = x;
            if (z_img) {
                const float z = __fmul_rn(__fsub_rn(x, shift_f[d]), inv_scale_f[d]);
                if (!(fabsf(z) < zb)) bits |= kScoreStatsBeyondZb;
                z_img[(size_t)d * pitch + e] = z;
            }
        }
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    if (bits && threadIdx.x == 0) atomicOr(flag, bits);
}

}  // namespace gmm
