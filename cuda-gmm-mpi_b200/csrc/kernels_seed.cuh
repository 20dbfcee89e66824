// kernels_seed.cuh — k-means++ seeding and the Lloyd assignment of gmm_seed_kmeans, for sm_90a.
//
// All kernels read the resident SoA copy xs [D][pitch] (coalesced per dimension).  Every sum that feeds a result is
// formed in a fixed order: per block of a CONSTANT number of events (not derived from the SM count), then block by
// block on the host.  No atomics, so a rerun is bit-identical.
//   d2    : [n] double, squared distance of each event to the nearest centre chosen so far
//   d(x,c): sum over d = 0 .. D-1 of (double(x_d) - double(c_d))^2, formed with __dsub_rn / __dmul_rn / __dadd_rn in
//           dimension order (no FMA contraction): a sequential float64 loop in numpy gives the same bits.
#pragma once
#include <cuda_runtime.h>
#include "kernels_simt.cuh"

namespace gmm {

constexpr int kSeedThreads = 256;
constexpr int kSeedBlockEvents = 1024;      // events per block of the k-means++ kernels: fixes the order of every sum
constexpr int kSeedMaxCand = 8;             // L = 2 + floor(ln K) candidates per round: 8 at K = 512
constexpr int kAssignThreads = 256;         // one event per thread, so kAssignThreads events per block
constexpr int kAssignSmemFloats = 8192;     // centre tile of the assignment: floor(8192 / D) centres (32 KB)

// One k-means++ target on the rank that owns it: scan `block` from the running prefix `start` for the first event whose
// inclusive prefix exceeds `target` (target = +inf: the last event of the block with d2 > 0).  block < 0: not here.
struct SeedPick {
    int block, pad;
    double start, target;
};

template <int D>
__device__ __forceinline__ double seed_dist(const float (&x)[D], const float* c) {
    double s = 0.0;
#pragma unroll
    for (int d = 0; d < D; d++) {
        const double t = __dsub_rn((double)x[d], (double)c[d]);
        s = __dadd_rn(s, __dmul_rn(t, t));
    }
    return s;
}

// d2 <- d(x, centre) (first) or min(d2, d(x, centre)), and the block's sum of d2 added event by event in index order
// (events past n add 0): bsum[block].
template <int D>
__global__ void __launch_bounds__(kSeedThreads)
kmeanspp_update_kernel(const float* __restrict__ xs, size_t pitch, int n, const float* __restrict__ centre, int first,
                       double* __restrict__ d2, double* __restrict__ bsum) {
    __shared__ float sc[D];
    __shared__ double sd[kSeedBlockEvents];
    if (threadIdx.x < D) sc[threadIdx.x] = centre[threadIdx.x];
    __syncthreads();
    const int base = blockIdx.x * kSeedBlockEvents;
    for (int j = threadIdx.x; j < kSeedBlockEvents; j += kSeedThreads) {
        const int e = base + j;
        double v = 0.0;
        if (e < n) {
            float x[D];
#pragma unroll
            for (int d = 0; d < D; d++) x[d] = xs[(size_t)d * pitch + e];
            v = seed_dist<D>(x, sc);
            if (!first) v = fmin(d2[e], v);
            d2[e] = v;
        }
        sd[j] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int j = 0; j < kSeedBlockEvents; j++) s = __dadd_rn(s, sd[j]);
        bsum[blockIdx.x] = s;
    }
}

// Potential of each of the L candidate centres cand [L][D]: sum of min(d2, d(x, c_l)) per block into bpot [block][8]
// (each thread adds its events in order, then a fixed shuffle tree per warp, then the warps in order).  d2 is not written.
template <int D>
__global__ void __launch_bounds__(kSeedThreads)
kmeanspp_potential_kernel(const float* __restrict__ xs, size_t pitch, int n, const float* __restrict__ cand, int L,
                          const double* __restrict__ d2, double* __restrict__ bpot) {
    __shared__ float sc[kSeedMaxCand * D];
    __shared__ double sp[kSeedMaxCand][kSeedThreads];       // the thread's running sums (registers would spill at D = 32)
    __shared__ double sw[kSeedThreads / 32][kSeedMaxCand];
    for (int i = threadIdx.x; i < L * D; i += kSeedThreads) sc[i] = cand[i];
    for (int l = 0; l < kSeedMaxCand; l++) sp[l][threadIdx.x] = 0.0;
    __syncthreads();
    const int base = blockIdx.x * kSeedBlockEvents;
    for (int j = threadIdx.x; j < kSeedBlockEvents; j += kSeedThreads) {
        const int e = base + j;
        if (e >= n) break;
        float x[D];
#pragma unroll
        for (int d = 0; d < D; d++) x[d] = xs[(size_t)d * pitch + e];
        const double m = d2[e];
#pragma unroll 1
        for (int l = 0; l < L; l++) sp[l][threadIdx.x] = __dadd_rn(sp[l][threadIdx.x], fmin(m, seed_dist<D>(x, sc + l * D)));
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int l = 0; l < kSeedMaxCand; l++) {
        const double s = warp_sum(sp[l][threadIdx.x]);
        if (lane == 0) sw[warp][l] = s;
    }
    __syncthreads();
    if (threadIdx.x < L) {
        double s = 0.0;
        for (int w = 0; w < kSeedThreads / 32; w++) s += sw[w][threadIdx.x];
        bpot[(size_t)blockIdx.x * kSeedMaxCand + threadIdx.x] = s;
    }
}

// One CTA (one warp) per target: the sequential scan of SeedPick, then the chosen event's row -> cand [target][D] and its
// local index -> idx [target].  Rows of targets another rank owns are left as they are (zeros).
__global__ void __launch_bounds__(32)
kmeanspp_pick_kernel(const double* __restrict__ d2, int n, const SeedPick* __restrict__ picks, const float* __restrict__ x_aos,
                     int D, float* __restrict__ cand, int* __restrict__ idx) {
    const SeedPick p = picks[blockIdx.x];
    if (p.block < 0) return;
    __shared__ int found;
    if (threadIdx.x == 0) {
        const int e0 = p.block * kSeedBlockEvents, e1 = min(n, e0 + kSeedBlockEvents);
        double run = p.start;
        int hit = -1, last = -1;
        for (int e = e0; e < e1; e++) {
            const double v = d2[e];
            run = __dadd_rn(run, v);
            if (v > 0.0) last = e;
            if (run > p.target) { hit = e; break; }
        }
        found = hit >= 0 ? hit : last;
        idx[blockIdx.x] = found;
    }
    __syncthreads();
    if (found >= 0 && threadIdx.x < D) cand[blockIdx.x * D + threadIdx.x] = x_aos[(size_t)found * D + threadIdx.x];
}

// Lloyd assignment: each event to the nearest of K centres [K][D] in FP32 (difference form, sum of (x - c)^2 with fused
// multiply-adds in dimension order; ties to the lowest k), centres staged through shared memory in tiles.  Writes the
// one-hot responsibilities memb [k][mpitch] for k < Kw (rows K .. Kw - 1 are zeros: the tensor M-step's 32-cluster boxes
// read them), the label, and per block the number of changed labels and the sum of the FP32 distances in double.
template <int D>
__global__ void __launch_bounds__(kAssignThreads)
kmeans_assign_kernel(const float* __restrict__ xs, size_t pitch, int n, const float* __restrict__ centres, int K, int Kw,
                     float* __restrict__ memb, size_t mpitch, int* __restrict__ labels, int* __restrict__ bchanged,
                     double* __restrict__ binertia) {
    constexpr int TILE = kAssignSmemFloats / D;
    __shared__ __align__(16) float sc[TILE * D];
    __shared__ double sw[kAssignThreads / 32];
    __shared__ int sn[kAssignThreads / 32];
    const int e = blockIdx.x * kAssignThreads + threadIdx.x;
    const bool valid = e < n;
    float x[D];
#pragma unroll
    for (int d = 0; d < D; d++) x[d] = valid ? xs[(size_t)d * pitch + e] : 0.0f;
    float best = INFINITY;
    int bk = 0;
    for (int k0 = 0; k0 < K; k0 += TILE) {
        const int kc = min(TILE, K - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < kc * D; i += kAssignThreads) sc[i] = centres[(size_t)k0 * D + i];
        __syncthreads();
        for (int k = 0; k < kc; k++) {
            const float* c = sc + k * D;
            float s = 0.0f;
#pragma unroll
            for (int d = 0; d < D; d++) {
                const float t = x[d] - c[d];
                s = fmaf(t, t, s);
            }
            if (s < best) { best = s; bk = k0 + k; }
        }
    }
    int changed = 0;
    double in = 0.0;
    if (valid) {
        for (int k = 0; k < Kw; k++) memb[(size_t)k * mpitch + e] = (k == bk) ? 1.0f : 0.0f;
        changed = labels[e] != bk ? 1 : 0;
        labels[e] = bk;
        in = (double)best;
    }
    in = warp_sum(in);
    changed = __reduce_add_sync(0xffffffffu, changed);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sw[warp] = in; sn[warp] = changed; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        int m = 0;
        for (int w = 0; w < kAssignThreads / 32; w++) { s += sw[w]; m += sn[w]; }
        binertia[blockIdx.x] = s;
        bchanged[blockIdx.x] = m;
    }
}

}  // namespace gmm
