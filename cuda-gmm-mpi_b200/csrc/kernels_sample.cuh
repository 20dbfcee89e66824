// kernels_sample.cuh — gmm_sample's kernel: events drawn from a Gaussian mixture, for sm_90a.
//
// Every event is a function of (parameters, seed, global index g) alone (the semantics are spelt out in gmm.h):
//   words   Philox4x32-10, key (lo32(seed), hi32(seed)), block j of event g at counter (lo32(g), hi32(g), j, 0)
//   label   u = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53; the first k with u T < C_k (C = cumulative pi in double, T = C_{K-1}),
//           or `klast` (the last cluster with pi > 0) when rounding leaves none
//   normals Box-Muller in float on words (2 + 2p, 3 + 2p)
//   event   x_d = mu_d + sum_{j >= d} U_dj z_j, fmaf in ascending j, U the upper-triangular factor of R = U U^T
// Parameter block (uploaded by the host per call): cum [K] double, padded to an even count, then one record of
// sample_rec_floats(D) floats per cluster: for d = 0 .. D-1 the row (mu_d, U_dd, .., U_d,D-1), then zero padding.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace gmm {

constexpr int kSampleThreads = 256;                 // one event per thread: a tile of 256 events per block iteration
constexpr int kSampleStageBytes = 110 * 1024;       // tile + parameters up to this size: parameters in shared memory, 2 blocks/SM

// floats per cluster record (a multiple of 4: records are 16-byte aligned and read as float4)
__host__ __device__ constexpr int sample_rec_floats(int D) { return (D + D * (D + 1) / 2 + 3) & ~3; }
// row stride of the output tile in shared memory: odd, so that a warp writing dimension d of its 32 rows hits 32 banks
__host__ __device__ constexpr int sample_tile_stride(int D) { return D | 1; }
__host__ __device__ constexpr size_t sample_tile_bytes(int D) { return sizeof(float) * kSampleThreads * sample_tile_stride(D); }
// doubles of the cumulative weights in the parameter block (even: the records after them stay 16-byte aligned)
__host__ __device__ constexpr int sample_cum_len(int K) { return (K + 1) & ~1; }
__host__ __device__ constexpr size_t sample_block_bytes(int K, int D) {
    return sizeof(double) * sample_cum_len(K) + sizeof(float) * (size_t)K * sample_rec_floats(D);
}

// Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11; the Random123 definition).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// u1 = ((float)a + 0.5f) 2^-32 in (0, 1], r = sqrtf(-2 logf(u1)) (at most ~6.8), (s, c) = sincospif((float)b 2^-31).
__device__ __forceinline__ void sample_box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    const float u1 = __fmul_rn(__fadd_rn(__uint2float_rn(a), 0.5f), 0x1p-32f);
    const float r = sqrtf(-2.0f * logf(u1));
    float s, c;
    sincospif(__fmul_rn(__uint2float_rn(b), 0x1p-31f), &s, &c);
    z0 = __fmul_rn(r, c);
    z1 = __fmul_rn(r, s);
}

__device__ __forceinline__ float f4_at(const float4& q, int i) { return i == 0 ? q.x : i == 1 ? q.y : i == 2 ? q.z : q.w; }

// Events [first, first + m) into out [m][D] (row-major) and labels [m].  stage = 1: the block copies the parameter
// block into shared memory behind the output tile (the caller sized the dynamic shared memory for it); 0: the records
// are read from global memory through L1.  Each block loops over tiles of kSampleThreads events: a thread forms its
// event's row in the tile, then the block writes the tile's rows to `out` as one contiguous, coalesced range.
template <int D>
__global__ void __launch_bounds__(kSampleThreads, 2)
sample_kernel(const double* __restrict__ block, int K, int klast, int stage, unsigned long long seed, long long first, int m,
              float* __restrict__ out, int* __restrict__ labels) {
    constexpr int REC = sample_rec_floats(D), S = sample_tile_stride(D), NP = (D + 1) / 2;
    extern __shared__ __align__(16) unsigned char sample_smem[];
    float* tile = reinterpret_cast<float*>(sample_smem);
    const double* cum = block;
    const float* recs = reinterpret_cast<const float*>(block + sample_cum_len(K));
    if (stage) {
        double* scum = reinterpret_cast<double*>(sample_smem + sample_tile_bytes(D));
        float4* srec = reinterpret_cast<float4*>(scum + sample_cum_len(K));
        const float4* grec = reinterpret_cast<const float4*>(recs);
        for (int i = threadIdx.x; i < K; i += kSampleThreads) scum[i] = cum[i];
        for (int i = threadIdx.x; i < K * (REC / 4); i += kSampleThreads) srec[i] = grec[i];
        __syncthreads();
        cum = scum;
        recs = reinterpret_cast<const float*>(srec);
    }
    const uint32_t key0 = (uint32_t)seed, key1 = (uint32_t)(seed >> 32);
    const double T = cum[K - 1];
    for (int t0 = blockIdx.x * kSampleThreads; t0 < m; t0 += gridDim.x * kSampleThreads) {
        const int i = t0 + threadIdx.x;
        if (i < m) {
            const unsigned long long g = (unsigned long long)(first + i);
            const uint32_t glo = (uint32_t)g, ghi = (uint32_t)(g >> 32);
            uint4 w = philox4x32_10(make_uint4(glo, ghi, 0u, 0u), key0, key1);
            const double u = (double)(((unsigned long long)(w.x >> 5) << 26) | (w.y >> 6)) * 0x1p-53;
            const double ut = __dmul_rn(u, T);
            int lo = 0, hi = K;                              // the first k with ut < cum[k], K if none
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (ut < cum[mid]) hi = mid; else lo = mid + 1;
            }
            const int k = lo < K ? lo : klast;
            labels[i] = k;
            float z[D];
#pragma unroll
            for (int p = 0; p < NP; p++) {                  // pair p: words 2 + 2p, 3 + 2p
                if (p & 1) w = philox4x32_10(make_uint4(glo, ghi, (uint32_t)((p + 1) / 2), 0u), key0, key1);
                float z0, z1;
                sample_box_muller((p & 1) ? w.x : w.z, (p & 1) ? w.y : w.w, z0, z1);
                z[2 * p] = z0;
                if (2 * p + 1 < D) z[2 * p + 1] = z1;
            }
            // the record streamed as float4, row by row: each x_d is finished (and leaves the registers) at the end of its
            // row.  Every index below is a constant once the loops are unrolled.
            const float4* r4 = reinterpret_cast<const float4*>(recs + (size_t)k * REC);
            float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int d = 0; d < D; d++) {
                const int e0 = d * (D + 1) - d * (d - 1) / 2;          // mu_d, then U_dd .. U_d,D-1
                if ((e0 & 3) == 0) q = r4[e0 >> 2];
                float x = f4_at(q, e0 & 3);
#pragma unroll
                for (int j = d; j < D; j++) {
                    const int e = e0 + 1 + (j - d);
                    if ((e & 3) == 0) q = r4[e >> 2];
                    x = fmaf(f4_at(q, e & 3), z[j], x);
                }
                tile[threadIdx.x * S + d] = x;
            }
        }
        __syncthreads();
        const int rows = min(kSampleThreads, m - t0);
        float* dst = out + (size_t)t0 * D;
        for (int j = threadIdx.x; j < rows * D; j += kSampleThreads) dst[j] = tile[(j / D) * S + j % D];
        __syncthreads();
    }
}

}  // namespace gmm
