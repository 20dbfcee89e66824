// kernels_combine.cuh — gmm_combine's device passes, for sm_90a: the entropy-criterion hierarchy of Baudry, Raftery,
// Celeux, Lo and Gottardo (2010) over the memberships the E-step leaves on the device, and the labels of a grouping.
//
// Merging groups A and B lowers the classification entropy -sum_n w_n sum_G tau_G ln tau_G by
//   dEnt(A, B) = sum_n w_n phi(tau_A(n), tau_B(n)),  phi(a, b) = (a+b) ln(a+b) - a ln a - b ln b.
// The kernels only read the [K][pitch] rows; a group's row tau_A is the float sum of its members' rows, formed on the fly
// in increasing component order.  Every sum has a fixed order and no atomics: a call's results are the same bits on every
// run with the same grid.
#pragma once
#include <cuda_runtime.h>

namespace gmm {

constexpr int kCombMaxK = 512;                          // GMM_MAX_CLUSTERS
constexpr int kCombTile = 32;                           // components per side of a pair tile
constexpr int kCombPairThreads = 256;
constexpr int kCombPairEvents = 64;                     // events a pair tile stages per iteration
constexpr int kCombStepThreads = 256;
constexpr int kCombStepEvents = 4 * kCombStepThreads;   // events per block of the step pass (one float4 per thread)
constexpr int kCombStepPerLane = kCombStepEvents / 128; // float4 per lane of a warp's group row
constexpr int kCombLabelThreads = 256;
constexpr int kCombSumThreads = 256;

// phi(a, b) as M h(m / M) with M = max, m = min and h(r) = (1 + r) log1p(r) - r ln r.  For r in (0, 1] both terms of h are
// >= 0, so nothing cancels, and M h <= 2 ln 2 M cannot overflow; phi = 0 when m = 0.
__device__ __forceinline__ float combine_phi(float a, float b) {
    const float M = fmaxf(a, b), m = fminf(a, b);
    if (!(m > 0.0f)) return 0.0f;
    const float r = m / M;
    return M * ((1.0f + r) * log1pf(r) - r * logf(r));
}

// Index of pair (a, b), a < b, in the row-major upper triangle of K components; the K masses follow the K(K-1)/2 pairs.
__host__ __device__ __forceinline__ int combine_pair_index(int a, int b, int K) { return a * (2 * K - a - 1) / 2 + (b - a - 1); }

// The all-pairs pass: every group a singleton.  blockIdx.x = tile pair (I <= J, row-major over the upper triangle of
// ceil(K / 32) tiles of 32 components), blockIdx.y = event range [y range_events, (y + 1) range_events) clipped to n
// (range_events a multiple of kCombPairEvents).  Each iteration stages the tiles' rows for 64 events in shared memory,
// transposed, with coalesced float4 loads; rows >= K and events >= n stage 0, which gives phi = 0 and mass 0.  Thread
// (lane, warp) owns pairs (32 I + lane, 32 J + warp + 8 j), j < 4, summed over events in order in double.  The diagonal
// tiles' warp 0 also sums the masses m_k = sum w tau_k.  partial[y][P] receives each pair and mass of the range once.
template <bool WEIGHTED>
__global__ void __launch_bounds__(kCombPairThreads)
combine_pairs_kernel(const float* __restrict__ memb, size_t pitch, int n, int K, const float* __restrict__ w, int range_events,
                     double* __restrict__ partial, int P) {
    __shared__ float sA[kCombPairEvents][kCombTile + 1];
    __shared__ float sB[kCombPairEvents][kCombTile + 1];
    __shared__ float sw[kCombPairEvents];
    const int T = (K + kCombTile - 1) / kCombTile;
    int t = blockIdx.x, I = 0;
    while (t >= T - I) { t -= T - I; I++; }
    const int J = I + t;
    const bool diag = I == J;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int e_begin = blockIdx.y * range_events, e_end = min(n, e_begin + range_events);
    constexpr int Q = kCombPairEvents / 4;
    double acc[4] = {0.0, 0.0, 0.0, 0.0}, mass = 0.0;
    float (*sb)[kCombTile + 1] = diag ? sA : sB;
    for (int e0 = e_begin; e0 < e_end; e0 += kCombPairEvents) {
        const int sides = diag ? 1 : 2;
        for (int i = threadIdx.x; i < sides * kCombTile * Q; i += kCombPairThreads) {
            const int side = i / (kCombTile * Q), r = (i / Q) % kCombTile, q = i % Q;
            const int k = (side ? J : I) * kCombTile + r, e = e0 + 4 * q;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < K && e < e_end) {
                v = __ldg(reinterpret_cast<const float4*>(memb + (size_t)k * pitch + e));
                if (e + 1 >= e_end) v.y = 0.f;
                if (e + 2 >= e_end) v.z = 0.f;
                if (e + 3 >= e_end) v.w = 0.f;
            }
            float (*s)[kCombTile + 1] = side ? sB : sA;
            s[4 * q][r] = v.x; s[4 * q + 1][r] = v.y; s[4 * q + 2][r] = v.z; s[4 * q + 3][r] = v.w;
        }
        if (WEIGHTED && threadIdx.x < kCombPairEvents) {
            const int e = e0 + threadIdx.x;
            sw[threadIdx.x] = e < e_end ? w[e] : 0.f;
        }
        __syncthreads();
#pragma unroll 2
        for (int e = 0; e < kCombPairEvents; e++) {
            const float va = sA[e][lane];
            double we = 1.0;
            if (WEIGHTED) we = (double)sw[e];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int bl = warp + 8 * j;
                if (!diag || lane < bl) {
                    const float ph = combine_phi(va, sb[e][bl]);
                    if (WEIGHTED) acc[j] = fma((double)ph, we, acc[j]);
                    else acc[j] += (double)ph;
                }
            }
            if (diag && warp == 0) {
                if (WEIGHTED) mass = fma((double)va, we, mass);
                else mass += (double)va;
            }
        }
        __syncthreads();
    }
    double* out = partial + (size_t)blockIdx.y * P;
    const int a = I * kCombTile + lane;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int b = J * kCombTile + warp + 8 * j;
        if (a < b && b < K) out[combine_pair_index(a, b, K)] = acc[j];
    }
    if (diag && warp == 0 && a < K) out[K * (K - 1) / 2 + a] = mass;
}

// out[j] = sum over ranges r in order of partial[r][j], j < P.
__global__ void __launch_bounds__(kCombSumThreads)
combine_sum_ranges_kernel(const double* __restrict__ partial, int ranges, int P, double* __restrict__ out) {
    for (int j = blockIdx.x * kCombSumThreads + threadIdx.x; j < P; j += gridDim.x * kCombSumThreads) {
        double s = 0.0;
        for (int r = 0; r < ranges; r++) s += partial[(size_t)r * P + j];
        out[j] = s;
    }
}

// Float sum of the rows members[b .. e) at float4 index q, left to right (an empty list gives 0).
__device__ __forceinline__ float4 combine_group_row(const float4* __restrict__ rows, size_t step, const int* members, int b, int e,
                                                   int q) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (b < e) v = __ldcs(rows + (size_t)members[b] * step + q);
    for (int i = b + 1; i < e; i++) {
        const float4 u = __ldcs(rows + (size_t)members[i] * step + q);
        v.x = __fadd_rn(v.x, u.x); v.y = __fadd_rn(v.y, u.y); v.z = __fadd_rn(v.z, u.z); v.w = __fadd_rn(v.w, u.w);
    }
    return v;
}

// The step pass: the gains of group g against every live group h != g, after g was formed by a merge.  The L live groups
// are members[goff[h] .. goff[h + 1]) (increasing components, goff[L] = K).  Blocks of kCombStepEvents events go to CTA
// blockIdx.x, + gridDim.x, ...: all threads form tau_g of the block (events >= n give 0, so phi = 0), then warp
// h mod 8 forms each tau_h from the original rows, and a warp's per-lane double sums are reduced in a fixed shuffle tree
// and added to the CTA's slot of h in block order.  One read of all K rows per pass.  partial[blockIdx.x][L]; slot g is 0.
template <bool WEIGHTED>
__global__ void __launch_bounds__(kCombStepThreads)
combine_step_kernel(const float* __restrict__ memb, size_t pitch, int n, const float* __restrict__ w, const int* __restrict__ members,
                    const int* __restrict__ goff, int L, int g, double* __restrict__ partial) {
    __shared__ int s_mem[kCombMaxK];
    __shared__ int s_off[kCombMaxK + 1];
    __shared__ double s_acc[kCombMaxK];
    __shared__ float4 s_g[kCombStepThreads];
    __shared__ float4 s_w[WEIGHTED ? kCombStepThreads : 1];
    const int K = goff[L];
    for (int i = threadIdx.x; i < K; i += kCombStepThreads) s_mem[i] = members[i];
    for (int i = threadIdx.x; i <= L; i += kCombStepThreads) s_off[i] = goff[i];
    for (int i = threadIdx.x; i < L; i += kCombStepThreads) s_acc[i] = 0.0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gb = s_off[g], ge = s_off[g + 1];
    const size_t step = pitch >> 2;
    const float4* rows = reinterpret_cast<const float4*>(memb);
    const int nq = (n + 3) >> 2;
    const int nblocks = (n + kCombStepEvents - 1) / kCombStepEvents;
    for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const int q0 = blk * kCombStepThreads;
        {
            const int q = q0 + threadIdx.x;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q < nq) {
                v = combine_group_row(rows, step, s_mem, gb, ge, q);
                const int e = 4 * q;                     // the rows' tail beyond n is not the memberships of any event
                if (e + 1 >= n) v.y = 0.f;
                if (e + 2 >= n) v.z = 0.f;
                if (e + 3 >= n) v.w = 0.f;
            }
            s_g[threadIdx.x] = v;
            if (WEIGHTED) s_w[threadIdx.x] = q < nq ? __ldg(reinterpret_cast<const float4*>(w) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncthreads();
        for (int h = warp; h < L; h += kCombStepThreads / 32) {
            if (h == g) continue;
            const int hb = s_off[h], he = s_off[h + 1];
            float4 t[kCombStepPerLane];
#pragma unroll
            for (int i = 0; i < kCombStepPerLane; i++) {
                const int q = q0 + lane + 32 * i;
                t[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (q < nq && hb < he) t[i] = __ldcs(rows + (size_t)s_mem[hb] * step + q);
            }
            for (int m = hb + 1; m < he; m++) {
                const float4* row = rows + (size_t)s_mem[m] * step;
#pragma unroll
                for (int i = 0; i < kCombStepPerLane; i++) {
                    const int q = q0 + lane + 32 * i;
                    if (q < nq) {
                        const float4 u = __ldcs(row + q);
                        t[i].x = __fadd_rn(t[i].x, u.x); t[i].y = __fadd_rn(t[i].y, u.y);
                        t[i].z = __fadd_rn(t[i].z, u.z); t[i].w = __fadd_rn(t[i].w, u.w);
                    }
                }
            }
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < kCombStepPerLane; i++) {
                const float4 G = s_g[lane + 32 * i];
                const float p0 = combine_phi(G.x, t[i].x), p1 = combine_phi(G.y, t[i].y);
                const float p2 = combine_phi(G.z, t[i].z), p3 = combine_phi(G.w, t[i].w);
                if (WEIGHTED) {
                    const float4 wv = s_w[lane + 32 * i];
                    s = fma((double)p0, (double)wv.x, s); s = fma((double)p1, (double)wv.y, s);
                    s = fma((double)p2, (double)wv.z, s); s = fma((double)p3, (double)wv.w, s);
                } else {
                    s += (double)p0; s += (double)p1; s += (double)p2; s += (double)p3;
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
            if (lane == 0) s_acc[h] += s;
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < L; i += kCombStepThreads) partial[(size_t)blockIdx.x * L + i] = s_acc[i];
}

// Labels of a grouping: per event, the group sums of members[goff[g] .. goff[g + 1]) for g < G, the first g of the
// largest sum (NaN sums skipped; -1 and NaN when every sum is NaN).  Four events per thread (one float4 of each row),
// grid-strided; labels and maxima to [pitch]-long buffers.
__global__ void __launch_bounds__(kCombLabelThreads)
combine_labels_kernel(const float* __restrict__ memb, size_t pitch, int n, const int* __restrict__ members, const int* __restrict__ goff,
                      int G, int* __restrict__ labels, float* __restrict__ maxv) {
    __shared__ int s_mem[kCombMaxK];
    __shared__ int s_off[kCombMaxK + 1];
    const int K = goff[G];
    for (int i = threadIdx.x; i < K; i += kCombLabelThreads) s_mem[i] = members[i];
    for (int i = threadIdx.x; i <= G; i += kCombLabelThreads) s_off[i] = goff[i];
    __syncthreads();
    const size_t step = pitch >> 2;
    const float4* rows = reinterpret_cast<const float4*>(memb);
    const int nq = (n + 3) >> 2;
    for (int q = blockIdx.x * kCombLabelThreads + threadIdx.x; q < nq; q += gridDim.x * kCombLabelThreads) {
        const float nan = __int_as_float(0x7fc00000);
        float4 best = make_float4(nan, nan, nan, nan);
        int4 lab = make_int4(-1, -1, -1, -1);
        for (int g = 0; g < G; g++) {
            const float4 v = combine_group_row(rows, step, s_mem, s_off[g], s_off[g + 1], q);
            if (v.x == v.x && (lab.x < 0 || v.x > best.x)) { best.x = v.x; lab.x = g; }
            if (v.y == v.y && (lab.y < 0 || v.y > best.y)) { best.y = v.y; lab.y = g; }
            if (v.z == v.z && (lab.z < 0 || v.z > best.z)) { best.z = v.z; lab.z = g; }
            if (v.w == v.w && (lab.w < 0 || v.w > best.w)) { best.w = v.w; lab.w = g; }
        }
        reinterpret_cast<int4*>(labels)[q] = lab;
        reinterpret_cast<float4*>(maxv)[q] = best;
    }
}

}  // namespace gmm
