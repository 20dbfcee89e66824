// kernels_vb.cuh — the one device pass of gmm_vb_em that no E- or M-step kernel covers, for sm_90a.
//
// The variational lower bound contains the responsibility entropy -sum_n w_n sum_k g_kn ln g_kn.  Recovering it from the
// packed statistics and the logits cancels (two sums of about n x 40 whose difference can be about 0), so it is read
// straight from the stored memberships: one coalesced, memory-bound pass of 4 K bytes per event.
#pragma once
#include <cuda_runtime.h>

namespace gmm {

constexpr int kEntropyThreads = 256;
constexpr int kEntropyBlocksPerSm = 4;

__device__ __forceinline__ double entropy_xlogx(float g) { return g > 0.0f ? (double)(g * logf(g)) : 0.0; }

// partial[blockIdx.x] = sum over this block's events e < n of w_e sum_{k<K} g ln g (0 ln 0 = 0; w_e = 1 without weights).
// memb: [>= K][pitch] cluster-major, pitch a multiple of 4 floats (rows 16-byte aligned).  Each thread takes groups of 4
// consecutive events (one float4 per row), grid-strided; per event the K terms are added in double in cluster order, the
// events of a thread in index order, then the warps in a fixed tree and the block's warps in order.  No atomics: the
// partials of a given grid are the same bits on every run; the caller adds them in block order.
template <bool WEIGHTED>
__global__ void __launch_bounds__(kEntropyThreads)
resp_entropy_kernel(const float* __restrict__ memb, size_t pitch, int n, int K, const float* __restrict__ w,
                    double* __restrict__ partial) {
    __shared__ double sw[kEntropyThreads / 32];
    const int nq = (n + 3) >> 2;
    const size_t step = pitch >> 2;
    double acc = 0.0;
    for (int q = blockIdx.x * kEntropyThreads + threadIdx.x; q < nq; q += gridDim.x * kEntropyThreads) {
        const float4* p = reinterpret_cast<const float4*>(memb) + q;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll 4
        for (int k = 0; k < K; k++) {
            const float4 g = __ldcs(p + (size_t)k * step);
            s0 += entropy_xlogx(g.x);
            s1 += entropy_xlogx(g.y);
            s2 += entropy_xlogx(g.z);
            s3 += entropy_xlogx(g.w);
        }
        const int e = 4 * q;                                 // the rows' tail beyond n is not the memberships of any event
        if (WEIGHTED) {
            const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + q);
            acc += (double)wv.x * s0;
            if (e + 1 < n) acc += (double)wv.y * s1;
            if (e + 2 < n) acc += (double)wv.z * s2;
            if (e + 3 < n) acc += (double)wv.w * s3;
        } else {
            acc += s0;
            if (e + 1 < n) acc += s1;
            if (e + 2 < n) acc += s2;
            if (e + 3 < n) acc += s3;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < kEntropyThreads / 32; i++) s += sw[i];
        partial[blockIdx.x] = s;
    }
}

}  // namespace gmm
