// kernels_multisample.cuh — the one device pass of gmm_em_multisample that no E- or M-step kernel covers, for sm_90a.
//
// Sample s is the event range [o_s, o_{s+1}); its components are shared, its mixing weights pi_{s,k} its own.  The
// library's E-step under the pooled weights pi_k gives r_nk ~ pi_k N(x_n | k), so with rho_{s,k} = pi_{s,k} / pi_k the
// per-sample posteriors are r'_nk = r_nk rho_{s,k} / S_n, S_n = sum_j r_nj rho_{s,j}, and ln p'(x_n) = ln p(x_n) + ln S_n.
// The reweight pass forms r' in place, the correction sum_n w_n ln S_n and the per-sample masses
// M_{s,k} = sum_{n in s} w_n r'_nk and n_s = sum_{n in s} w_n: one read and one write of every membership.
//
// Work units never cross a sample boundary: the host cuts the shard's events into windows of E events aligned to E and
// splits a window that holds a boundary into one unit per sample.  Persistent CTAs walk contiguous runs of units in
// order, accumulate the current sample's masses, and flush one partial record per (CTA, sample segment).  A finishing
// kernel adds the records of each sample in record order.  No atomics: a rerun on the same shard and grid gives the same
// bits.
#pragma once
#include <cuda_runtime.h>

namespace gmm {

constexpr int kMsThreads = 256;
constexpr int kMsWarps = kMsThreads / 32;
constexpr int kMsMaxSamples = 4096;
constexpr int kMsTileBytes = 64 * 1024;                 // shared-memory tile of K x E memberships at most
constexpr int kMsFinishThreads = 256;

// One unit: events [e0, e1) of sample s (shard-local indices), inside the window [e0 & ~(E - 1), + E); `part` is the
// partial record its (CTA, sample segment) flushes to.
struct MsUnit {
    int s, e0, e1, part;
};

// Events per window for K components: the largest power of two in [32, 256] with K E floats in kMsTileBytes.
__host__ __device__ inline int ms_window_events(int K) {
    int E = 256;
    while (E > 32 && (size_t)K * E * sizeof(float) > (size_t)kMsTileBytes) E >>= 1;
    return E;
}
__host__ __device__ inline size_t ms_smem_bytes(int K, int E, bool masses_only) {
    // tile [K][E] float | column sums [E] float | rho [K] float | masses [K] double | warp partials [2][kMsWarps] double
    const size_t tile = masses_only ? 0 : (size_t)K * E * sizeof(float) + (size_t)E * sizeof(float) + (size_t)K * sizeof(float);
    const size_t acc = (size_t)K * sizeof(double) + 2 * kMsWarps * sizeof(double);
    return ((tile + 15) & ~(size_t)15) + acc;
}

// Records [part][K + 2]: the K masses, then n_s (sum of the weights), then sum w ln S (0 in the masses-only mode).
// CTA b walks units [cta_begin[b], cta_begin[b + 1]).
//   MASSES_ONLY: rho = 1 for every sample; r' = r, nothing is written and nothing is added to the log-likelihood.
//   otherwise, per event of sample s: t_k = r_k * rho_{s,k}, S = t_0 + t_1 + ... in increasing k (one rounding per
//   operation, no contraction), r'_k = t_k / S, rows k < K and events of the unit only.
// The masses of a unit are summed per row by one warp (lane-strided float4s, events in order within a float4, then a fixed
// shuffle tree) and added to the CTA's accumulator unit after unit; n_s and the correction per thread, then a fixed tree.
template <bool WEIGHTED, bool MASSES_ONLY>
__global__ void __launch_bounds__(kMsThreads)
ms_reweight_kernel(float* __restrict__ memb, size_t pitch, int K, const float* __restrict__ w, const float* __restrict__ rho,
                   const MsUnit* __restrict__ units, const int* __restrict__ cta_begin, int E, double* __restrict__ partial) {
    extern __shared__ __align__(16) unsigned char ms_smem[];
    float* tile = reinterpret_cast<float*>(ms_smem);                       // [K][E]
    float* colS = tile + (MASSES_ONLY ? 0 : (size_t)K * E);                 // [E]
    float* srho = colS + (MASSES_ONLY ? 0 : E);                             // [K]
    const size_t tile_bytes = MASSES_ONLY ? 0 : ((size_t)K * E + E + K) * sizeof(float);
    double* acc = reinterpret_cast<double*>(ms_smem + ((tile_bytes + 15) & ~(size_t)15));   // [K]
    double* red = acc + K;                                                  // [2][kMsWarps]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int u_begin = cta_begin[blockIdx.x], u_end = cta_begin[blockIdx.x + 1];
    const int nq = E >> 2;
    for (int k = tid; k < K; k += kMsThreads) acc[k] = 0.0;
    __syncthreads();                                        // acc[k] is zeroed and accumulated by different warps
    double n_acc = 0.0, ll_acc = 0.0;
    for (int u = u_begin; u < u_end; u++) {
        const MsUnit un = units[u];
        const int base = un.e0 & ~(E - 1);
        if (!MASSES_ONLY) {
            if (u == u_begin || units[u - 1].s != un.s)
                for (int k = tid; k < K; k += kMsThreads) srho[k] = rho[(size_t)un.s * K + k];
            // the float4s of the window that hold events of the unit, rows k < K
            for (int i = tid; i < K * nq; i += kMsThreads) {
                const int k = i / nq, q = i - k * nq, e = base + 4 * q;
                if (e + 4 > un.e0 && e < un.e1)
                    *reinterpret_cast<float4*>(tile + (size_t)k * E + 4 * q) =
                        __ldcg(reinterpret_cast<const float4*>(memb + (size_t)k * pitch + e));
            }
            __syncthreads();
        }
        // per event: S in increasing k, the correction and the weight sum (thread j owns column j)
        for (int j = tid; j < E; j += kMsThreads) {
            const int e = base + j;
            if (e < un.e0 || e >= un.e1) continue;
            const float we = WEIGHTED ? __ldg(w + e) : 1.0f;
            n_acc += (double)we;
            if (!MASSES_ONLY) {
                float S = 0.0f;
                for (int k = 0; k < K; k++) S = __fadd_rn(S, __fmul_rn(tile[(size_t)k * E + j], srho[k]));
                colS[j] = S;
                ll_acc += (double)we * log((double)S);
            }
        }
        if (!MASSES_ONLY) __syncthreads();
        // per row: r' written back, the masses summed
        for (int k = warp; k < K; k += kMsWarps) {
            const float rk = MASSES_ONLY ? 1.0f : srho[k];
            float* row = memb + (size_t)k * pitch;
            double m = 0.0;
            for (int q = lane; q < nq; q += 32) {
                const int e = base + 4 * q;
                if (e + 4 <= un.e0 || e >= un.e1) continue;
                float4 v = MASSES_ONLY ? __ldcg(reinterpret_cast<const float4*>(row + e))
                                       : *reinterpret_cast<const float4*>(tile + (size_t)k * E + 4 * q);
                const bool in0 = e >= un.e0 && e < un.e1, in1 = e + 1 >= un.e0 && e + 1 < un.e1;
                const bool in2 = e + 2 >= un.e0 && e + 2 < un.e1, in3 = e + 3 >= un.e0 && e + 3 < un.e1;
                if (!MASSES_ONLY) {
                    const float* S = colS + 4 * q;
                    v.x = __fdiv_rn(__fmul_rn(v.x, rk), S[0]);
                    v.y = __fdiv_rn(__fmul_rn(v.y, rk), S[1]);
                    v.z = __fdiv_rn(__fmul_rn(v.z, rk), S[2]);
                    v.w = __fdiv_rn(__fmul_rn(v.w, rk), S[3]);
                    if (in0 && in3) *reinterpret_cast<float4*>(row + e) = v;
                    else {                                       // a float4 shared with the neighbouring unit
                        if (in0) row[e] = v.x;
                        if (in1) row[e + 1] = v.y;
                        if (in2) row[e + 2] = v.z;
                        if (in3) row[e + 3] = v.w;
                    }
                }
                float4 wv = make_float4(1.f, 1.f, 1.f, 1.f);
                if (WEIGHTED) wv = __ldg(reinterpret_cast<const float4*>(w + e));
                if (in0) m += (double)wv.x * (double)v.x;
                if (in1) m += (double)wv.y * (double)v.y;
                if (in2) m += (double)wv.z * (double)v.z;
                if (in3) m += (double)wv.w * (double)v.w;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m += __shfl_down_sync(0xffffffffu, m, o);
            if (lane == 0) acc[k] += m;
        }
        // flush at the end of the CTA's sample segment
        if (u + 1 == u_end || units[u + 1].part != un.part) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                n_acc += __shfl_down_sync(0xffffffffu, n_acc, o);
                ll_acc += __shfl_down_sync(0xffffffffu, ll_acc, o);
            }
            if (lane == 0) { red[warp] = n_acc; red[kMsWarps + warp] = ll_acc; }
            __syncthreads();
            double* rec = partial + (size_t)un.part * (K + 2);
            for (int k = tid; k < K; k += kMsThreads) { rec[k] = acc[k]; acc[k] = 0.0; }
            if (tid == 0) {
                double sn = 0.0, sl = 0.0;
#pragma unroll
                for (int i = 0; i < kMsWarps; i++) { sn += red[i]; sl += red[kMsWarps + i]; }
                rec[K] = sn;
                rec[K + 1] = sl;
            }
            n_acc = ll_acc = 0.0;
        }
        __syncthreads();
    }
}

// out[s][j] = sum over the records [sample_part[s], sample_part[s + 1]) in order of record[j], j <= K (K masses, then
// n_s; 0 for a sample without records).  ll != NULL: thread 0 of block 0 adds the corrections of all records, in record
// order, to *ll (the log-likelihood slot of the statistics, before their all-reduce).
__global__ void __launch_bounds__(kMsFinishThreads)
ms_finish_kernel(const double* __restrict__ partial, const int* __restrict__ sample_part, int S, int K, double* __restrict__ out,
                 double* ll) {
    const int per = K + 1;
    for (int i = blockIdx.x * kMsFinishThreads + threadIdx.x; i < S * per; i += gridDim.x * kMsFinishThreads) {
        const int s = i / per, j = i - s * per;
        double v = 0.0;
        for (int p = sample_part[s]; p < sample_part[s + 1]; p++) v += partial[(size_t)p * (K + 2) + j];
        out[i] = v;
    }
    if (ll && blockIdx.x == 0 && threadIdx.x == 0) {
        double c = 0.0;
        for (int p = 0; p < sample_part[S]; p++) c += partial[(size_t)p * (K + 2) + K + 1];
        *ll += c;
    }
}

}  // namespace gmm
