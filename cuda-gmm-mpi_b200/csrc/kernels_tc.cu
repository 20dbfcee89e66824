// kernels_tc.cu — warpgroup-MMA (wgmma) kernels of the EM hot path for sm_90a.
//
// M-step (mstep_N + mstep_means + mstep_covariance1 of the reference,
// gaussian_kernel.cu:522-677) as ONE tensor-core contraction over the events:
//
//     S^T[f][k] = sum_n  phi_f(z_n) * g[k][n]        z = (x - shift) * inv_scale
//
// with the per-event feature vector phi = [1, z_d, z_i z_j (i>=j)] (F = 1+D+D(D+1)/2
// rows, shared by all clusters) as the A operand and the responsibilities as the
// B operand; FP32 accumulation in registers.
//
// Operand arithmetic.  The tensor cores' FP32 accumulation does not round to nearest — but it is EXACT as long as
// every partial sum is a multiple of one quantum and fits 24 bits.  The operands are therefore split into a
// FIXED-POINT leading part and a small remainder:
//     phi_f = ph + pl,   ph = q_f * round(phi_f / q_f),   |ph| <= 2^11 q_f     (q_f: power of two per feature row,
//                                                                              from the data's largest |z_d|)
//     g     = gh + gl,   gh = 2^-6 * round(2^6 g)   (0 .. 64 quanta)
// (both by a magic-number add: no conversion round trip), and the products go to two accumulator column groups
// per feature tile:
//     columns [0, 32):    sum ph * gh                 — every product a multiple of q_f 2^-6, at most 2^17 quanta;
//                                                       128 events per chain: <= 2^24 quanta: NO rounding at all
//     columns [32, 64):   sum ph * gl + pl * gs       — gs = g rounded once to FP16 (11 bits RELATIVE): with gh alone
//                                                       the dropped pl * gl would be O(pl / phi) of every event whose
//                                                       g is below the quantum; ~1 % of the magnitude, its truncation
//                                                       bias is 1e-8 of the statistic
// The raw-moment cancellation |mu - shift|^2 / sigma^2 ~ 100 multiplies unbiased rounding noise only.
// Each column group is its own N = NCL accumulator (NCL = 32 or 64 clusters per CTA): ph x gh into the exact one, then
// ph x gl and pl x gs into the remainder one.  All MMAs of a consumer have the same shape and no two accumulators overlap,
// so ptxas keeps the wgmma of a sub-tile in flight together (an N = 64 MMA filling both groups plus an N = 32 MMA into
// its upper half made it wait for every MMA before issuing the next, C7511).
//
// Dataflow per CTA (persistent over a contiguous range of events; NCL clusters and, at NCL = 64, half of the feature rows):
//   warp 0      TMA producer: tile [D][32 events] of the pre-standardised SoA copy z and raw responsibility boxes
//               [32 clusters][32 events] (2-D tensor maps, both SWIZZLE_128B, zero fill out of bounds)
//   warps 1-3   split the responsibilities and write the wgmma B images gh / gl / gs (no-swizzle core-matrix layout)
//   warpgroups 1 .. MT  consumers: each thread builds the A fragments of its feature rows (mstep_rows.h) from the raw z
//               tile in registers — the feature operand never goes through shared memory — and per 32 events the
//               warpgroup issues 2 x 3 wgmma per 64-row half it owns (A from registers: m64n32k16 for both halves of a
//               tile, or m64n64k16 for one half), each group running while the next is built.  The exact group is drained
//               every 128 events and the remainder group every 512 into FP32 round-to-nearest partial sums held in shared
//               memory (one private slot per thread), written ONCE per CTA (no scratch zeroing, no atomics).
// A second tiny kernel reduces the per-CTA partials in double and un-scales.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#if defined(__F16C__) && defined(__AVX__)
#include <immintrin.h>
#endif
#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "cuda_owned.h"
#include "host_math.h"
#include "kernels_tc.cuh"
#include "mstep_rows.h"
#include "tc_ptx.cuh"

namespace gmm {

using namespace ptx;

// ---------------------------------------------------------------------------
// M-step kernel configuration
// ---------------------------------------------------------------------------
constexpr int kTE = 32;          // events per sub-tile (MMA K extent per operand part)
constexpr int kNCL = 32;         // clusters per responsibility TMA box and per column block of the partial sums
constexpr int kNST = 3;          // responsibility operand stages
constexpr int kNRAW = 4;         // raw (TMA) stages
constexpr int kChunkSub = 4;     // sub-tiles per chain of the exact column group: 128 events (the bit budget below)
constexpr int kChunkSub2 = 16;   // sub-tiles per chain of the remainder column group (no exactness to protect: drained 4x less often)
// Bit budget of the exact accumulator: 11 (ph, every integer up to 2048 is an FP16 value) + 6 (gh) + 7 (128 events) = 24.
// The split favours phi: the remainder pl is rounded to FP16 RELATIVE to itself, so its (unbiased) rounding noise scales
// with the quantum of ph — on covariance entries 6e-6 per call with 9 + 8 bits, 1.2e-6 with 11 + 6 (scripts/emu_mstep.py).
constexpr int kPhiBits = 11;     // |ph| <= 2^11 quanta
constexpr float kGammaScale = 1024.0f;               // responsibilities are scaled by 2^10 in the operand
constexpr float kGammaMagic = 1.5f * 134217728.0f;   // 1.5 * 2^27: ulp = 16 = 2^-6 in the scaled units

// Row layout of the feature operand: mstep_rows.h.  Every operand row is a product z_a * z_b of two factors (a dimension
// or the ones pseudo-dimension); consumer thread (warp w, lane group gid) of tile mt owns the 4 rows
// mt * 128 + h * 64 + 16 w + gid + 8 s, which share the factor a.  The thread builds the wgmma A fragments of its rows
// from the raw z tile itself (register operand), so the feature operand never goes through shared memory.
//
// Two schedules, chosen by K (launch_mstep_d), with the same MT consumer warpgroups and 64 accumulators per thread:
//   NCL = 32  (K <= 32)  a CTA covers all 2 MT feature halves for 32 clusters: each consumer owns both halves of its tile
//   NCL = 64  (K > 32)   the two CTAs of an event range split the 2 MT halves, each for 64 clusters: each consumer owns one
//                        half (part p, consumer c: half p MT + c).  The feature operand of an event is built once per 64
//                        clusters instead of once per 32, and the pair shares its z / gamma tiles through L2.
template <int D, int NCL_> struct MCfg {
    static_assert(D % 4 == 0, "tensor M-step: D must be a multiple of 4");
    static_assert(NCL_ == 32 || NCL_ == 64, "tensor M-step: 32 or 64 clusters per CTA");
    static constexpr int NCL = NCL_;
    static constexpr int HPC = 64 / NCL;                  // 64-row feature halves per consumer warpgroup
    static constexpr int F = 1 + D + D * (D + 1) / 2;
    static constexpr int S = D / 4;
    static constexpr int MT = (4 * ((1 + 2 * S + S * (D / 2) + 7) / 8) * 8 + 127) / 128;   // feature tiles (mstep_tiles)
    static constexpr int G_PART = NCL * kTE * 2;
    static constexpr int G_STAGE = 3 * G_PART;            // gh, gl, gs: three K-major N = NCL images
    // raw z stage: the [D][32 events] tile (SWIZZLE_128B), padded to 1 KB, then 1 KB of ones (8 rows of the same swizzle:
    // the ones pseudo-dimension at a stage-relative address like every dimension)
    static constexpr int RAWZ = (D * kTE * 4 + 1023) / 1024 * 1024;
    static constexpr int RAWX = RAWZ + 1024;
    static constexpr int RAWG = NCL * kTE * 4;            // NCL / 32 boxes of [32 clusters][32 events]
    static constexpr int OFF_G = 0;
    static constexpr int OFF_RAWX = OFF_G + kNST * G_STAGE;
    static constexpr int OFF_RAWG = OFF_RAWX + kNRAW * RAWX;
    static constexpr int NCT = MT * 128;                  // consumer threads (one warpgroup per 128-row feature tile)
    static constexpr int OFF_RACC = OFF_RAWG + kNRAW * RAWG;   // [32][NCT] FP32 partial sums, one private column per thread
    static constexpr int OFF_BAR = OFF_RACC + 32 * NCT * 4;
    static constexpr int SMEM_BYTES = OFF_BAR + 512;
    static constexpr int THREADS = 128 + NCT;             // producer warpgroup, consumers
    // register pools: producer warpgroup / consumers.  The kernel is launched with REG_LAUNCH registers per thread
    // (the __launch_bounds__ maximum, which ptxas uses when setmaxnreg is present); setmaxnreg only redistributes that
    // allocation, so a warpgroup's increase waits until the others' decreases have freed enough — the sum must fit.
    // With one feature tile (256 threads) every thread may have 255 registers: no redistribution.
    static constexpr int REG_LAUNCH = (65536 / THREADS) / 8 * 8 > 255 ? 255 : (65536 / THREADS) / 8 * 8;
    static constexpr int REG_P = MT == 1 ? REG_LAUNCH : 56;
    static constexpr int REG_C = MT == 3 ? 152 : (MT == 2 ? 224 : REG_LAUNCH);
    static_assert(128 * REG_P + NCT * REG_C <= THREADS * REG_LAUNCH, "register pools");
    static_assert(OFF_RAWX % 1024 == 0 && RAWX % 1024 == 0 && RAWZ % 1024 == 0, "SWIZZLE_128B TMA destinations need 1024-byte alignment");
    static_assert(OFF_RAWG % 1024 == 0 && RAWG % 1024 == 0, "SWIZZLE_128B TMA destinations need 1024-byte alignment");
    static_assert(MT <= 3, "feature tiles");
};

template <int R, int L>
__device__ __forceinline__ void set_regs() {
    if constexpr (R < L) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
    else if constexpr (R > L) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// Rounding constants: (v + magic) - magic = q * round(v / q) with magic = 1.5 * 2^23 * q.  One quantum for the
// coordinate rows and one for the product rows (bound = the largest |z_d| of the data over ALL dimensions, rounded up
// to a power of two: after the standardisation the dimensions have the same scale).
struct MMagic { float lin, prod; };

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
    return v;
}

// Leading part / remainder of the feature a * b with rounding constant m: the product rows' operations of the staged
// layout for every row — a linear row is z_a * 1 (fma(z, 1, m) - m and fma(z, 1, -h) round as (z + m) - m and z - h),
// the constant row is 1 * 1 with m = 0.  Both parts come from the EXACT product, rounded once each.
__device__ __forceinline__ void feature_split(float a, float b, float m, float& h, float& l) {
    h = __fsub_rn(__fmaf_rn(a, b, m), m);
    l = __fmaf_rn(a, b, -h);
}

// Timing variants for scripts/prof_mstep.py (`make variant DEFS=-DGMM_MSTEP_CUT=n`); the default build is 0.
//   1  no MMAs: loads and operand build only (the fragments are kept alive, the stages released at the same points; with
//      no wgmma to wait on, the raw stage may be released before its loads land)
//   2  no feature build: the MMAs read the raw z words as their A fragments
//   3  no drains: the accumulators are added to the partial sums once, after the last sub-tile
// The results of a variant are wrong.
#ifndef GMM_MSTEP_CUT
#define GMM_MSTEP_CUT 0
#endif

// A fragments of one 64-row half: rows s = 0, 1 of the thread (slot 2h + s), events 16 ks + 2 qd + {0, 1, 8, 9}.
// za / zb*: the 8 events of the thread ([pair p] = events 8p + 2qd, +1); hi / lo [ks][4]: a0..a3 of k-step ks.
__device__ __forceinline__ void build_half(const float2 (&za)[4], const float2 (&zb0)[4], const float2 (&zb1)[4], float m0, float m1,
                                           uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
    for (int p = 0; p < 4; p++) {
        const int ks = p >> 1, u = p & 1;                      // a0 / a1: pair 2ks (rows s = 0, 1); a2 / a3: pair 2ks + 1
#if GMM_MSTEP_CUT == 2
        hi[ks][2 * u] = __float_as_uint(zb0[p].x); hi[ks][2 * u + 1] = __float_as_uint(zb1[p].x);
        lo[ks][2 * u] = __float_as_uint(zb0[p].y); lo[ks][2 * u + 1] = __float_as_uint(zb1[p].y);
        (void)za; (void)m0; (void)m1;
#else
        float h0, l0, h1, l1, h2, l2, h3, l3;
        feature_split(za[p].x, zb0[p].x, m0, h0, l0);
        feature_split(za[p].y, zb0[p].y, m0, h1, l1);
        feature_split(za[p].x, zb1[p].x, m1, h2, l2);
        feature_split(za[p].y, zb1[p].y, m1, h3, l3);
        hi[ks][2 * u] = pack_half2(h0, h1);                    // exact: <= 2048 quanta
        hi[ks][2 * u + 1] = pack_half2(h2, h3);
        lo[ks][2 * u] = pack_half2(l0, l1);
        lo[ks][2 * u + 1] = pack_half2(l2, l3);
#endif
    }
}

// The 8 events of one z-tile row (stage-relative swizzled address: chunk c of row r at c ^ (r & 7), see mstep_rows.h)
__device__ __forceinline__ void load_row(uint32_t addr, float2 (&z)[4]) {
#pragma unroll
    for (int p = 0; p < 4; p++) z[p] = lds_f2(addr ^ (uint32_t)(p << 5));
}

// The MMAs of one half (both k-steps) for NCL clusters: ph gh into the exact group, ph gl + pl gs into the remainder group.
template <int NCL>
__device__ __forceinline__ void issue_half(float (&ex)[NCL / 2], float (&rm)[NCL / 2], const uint32_t (&hi)[2][4], const uint32_t (&lo)[2][4],
                                           uint32_t gam, bool new1, bool new2) {
#pragma unroll
    for (int ks = 0; ks < kTE / 16; ks++) {
        const uint64_t hdesc = make_smem_desc(gam + ks * 256, /*LBO*/ 128, /*SBO*/ 512);     // gh
        const uint64_t ldesc = make_smem_desc(gam + NCL * kTE * 2 + ks * 256, 128, 512);     // gl
        const uint64_t sdesc = make_smem_desc(gam + 2 * NCL * kTE * 2 + ks * 256, 128, 512); // gs
#if GMM_MSTEP_CUT == 1
        asm volatile("" ::"r"(hi[ks][0]), "r"(hi[ks][1]), "r"(hi[ks][2]), "r"(hi[ks][3]), "r"(lo[ks][0]), "r"(lo[ks][1]), "r"(lo[ks][2]),
                     "r"(lo[ks][3]), "l"(hdesc), "l"(ldesc), "l"(sdesc));
        (void)ex; (void)rm; (void)new1; (void)new2;
#else
        if constexpr (NCL == 32) {
            wgmma_m64n32k16_rs(ex, hi[ks][0], hi[ks][1], hi[ks][2], hi[ks][3], hdesc, ks > 0 || !new1);   // ph gh
            wgmma_m64n32k16_rs(rm, hi[ks][0], hi[ks][1], hi[ks][2], hi[ks][3], ldesc, ks > 0 || !new2);   // ph gl
            wgmma_m64n32k16_rs(rm, lo[ks][0], lo[ks][1], lo[ks][2], lo[ks][3], sdesc, true);              // + pl gs
        } else {
            wgmma_m64n64k16_rs(ex, hi[ks][0], hi[ks][1], hi[ks][2], hi[ks][3], hdesc, ks > 0 || !new1);
            wgmma_m64n64k16_rs(rm, hi[ks][0], hi[ks][1], hi[ks][2], hi[ks][3], ldesc, ks > 0 || !new2);
            wgmma_m64n64k16_rs(rm, lo[ks][0], lo[ks][1], lo[ks][2], lo[ks][3], sdesc, true);
        }
#endif
    }
}

// Feature tile `mt` is drained after sub-tile i when its 128-event chain ends there: the chains of the tiles are
// staggered by one sub-tile each, so that the consumer warpgroups do not all drain after the same sub-tile.
// The remainder column group rides along and is drained (and restarted) only at every fourth of those points.
__device__ __forceinline__ bool chain_ends(int i, int mt, int nsub) { return ((i + mt) % kChunkSub) == kChunkSub - 1 || i == nsub - 1; }
__device__ __forceinline__ bool chain_starts(int i, int mt) { return i == 0 || ((i + mt) % kChunkSub) == 0; }
__device__ __forceinline__ bool chain2_ends(int i, int mt, int nsub) { return ((i + mt) % kChunkSub2) == kChunkSub2 - 1 || i == nsub - 1; }
__device__ __forceinline__ bool chain2_starts(int i, int mt) { return i == 0 || ((i + mt) % kChunkSub2) == 0; }

// opmap[row] = a | b << 8: the operand factors of row `row` (mstep_row_layout; codes >= kRowOne: rows of the ones block).
// Grid (ranges * 64 / NCL, ceil(K / NCL)): CTA x = range * 64 / NCL + part, so with NCL = 64 the two CTAs of a range run in
// the same wave and the second reader of every z / gamma tile finds it in L2.
// WT (gmm_set_weights): the responsibility operand is g * w^, w^ = 1 for w = w_max (the largest weight), else w * w_inv
// (w_inv = 1 / w_max rounded; no division in the 56-register pool), so w^ is at most 1 and the product lies in [0, 1] like g:
// the split below and its bit budget are unchanged.  The library runs this instance for weights of one positive value only
// (gmm_api.cu kWeightRangeTc), where w^ is exactly 0 or 1 and the operand is the unweighted one with rows removed.  wts: [>= 32 * ceil(n / 32)] floats, zero beyond n.
// mstep_tc_finalize_kernel multiplies the sums by w_max.
template <int D, int NCL, bool WT = false>
__global__ void __launch_bounds__(MCfg<D, NCL>::THREADS, 1)
mstep_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_g, int n, int K,
                float* __restrict__ scratch, int events_per_cta, const __grid_constant__ MMagic magic, const int* __restrict__ opmap,
                const float* __restrict__ wts, float w_max, float w_inv) {
    using C = MCfg<D, NCL>;
    constexpr int HPC = C::HPC;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
    uint64_t* raw_full = bars;                 // [kNRAW]
    uint64_t* raw_empty = bars + kNRAW;        // [kNRAW]
    uint64_t* op_full = bars + 2 * kNRAW;      // [kNST]
    uint64_t* op_empty = op_full + kNST;       // [kNST]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int range = blockIdx.x / (2 / HPC), part = blockIdx.x % (2 / HPC);
    const int e_begin = range * events_per_cta;
    const int e_end = min(n, e_begin + events_per_cta);
    const int nsub = (e_end - e_begin + kTE - 1) / kTE;
    const int k0 = blockIdx.y * NCL;

    // ---- one-time setup: the ones block of every raw stage, barriers ----
    for (int i = threadIdx.x; i < kNRAW * 256; i += C::THREADS)
        reinterpret_cast<float*>(smem + C::OFF_RAWX + (i >> 8) * C::RAWX + C::RAWZ)[i & 255] = 1.0f;
    if (threadIdx.x == 0) {
        // raw stage: 3 responsibility-splitting warps and every consumer warp load from it
        for (int s = 0; s < kNRAW; s++) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], 3 + 4 * C::MT); }
        for (int s = 0; s < kNST; s++) { mbar_init(&op_full[s], 3); mbar_init(&op_empty[s], 4 * C::MT); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        set_regs<C::REG_P, C::REG_LAUNCH>();
        if (warp == 0) {
            // ===================== TMA producer =====================
            // one responsibility box per 32 clusters that holds a live one (a box wholly above K is not loaded: the
            // columns it would fill are not read back)
            const int nbox = min(NCL, K - k0 + kNCL - 1) / kNCL;
            if (elect_one()) {
                for (int i = 0; i < nsub; i++) {
                    const int st = i % kNRAW, ph = (i / kNRAW) & 1;
                    mbar_wait_parked(&raw_empty[st], ph ^ 1, 500);
                    mbar_arrive_expect_tx(&raw_full[st], kTE * D * 4 + nbox * kNCL * kTE * 4);
                    const int e0 = e_begin + i * kTE;
                    tma_load_2d(smem + C::OFF_RAWX + st * C::RAWX, &tm_x, e0, 0, &raw_full[st]);
                    for (int b = 0; b < nbox; b++)
                        tma_load_2d(smem + C::OFF_RAWG + st * C::RAWG + b * kNCL * kTE * 4, &tm_g, e0, k0 + b * kNCL, &raw_full[st]);
                }
            }
        } else {
            // ===================== responsibility operand: warps 1-3 =====================
            // item (cluster row k, 8-event chunk ce): 4 NCL per sub-tile, thread bt takes bt, bt + 96, ...
            // The raw tile is written by TMA with SWIZZLE_128B (16-byte chunk c of row r sits at chunk c ^ (r & 7)), so
            // 8 lanes reading the same chunk of 8 consecutive rows hit 8 different bank groups; the operand image puts
            // the 4 K-chunks of an 8-row group next to each other (LBO = 128, SBO = 512), so a warp stores 512
            // contiguous bytes: no bank conflicts either way.  Each item's images are stored before the next is split,
            // so the 56-register pool holds one item at a time.
            const int bt = threadIdx.x - 32;
            constexpr int NITEM = 4 * NCL, NIT = (NITEM + 95) / 96;
            for (int i = 0; i < nsub; i++) {
                const int rs = i % kNRAW, rph = (i / kNRAW) & 1;
                const int os = i % kNST, oph = (i / kNST) & 1;
                // every item of this thread has the 8-event chunk ce = (bt & 31) >> 3 (items step by 96): its 8 weights are
                // loaded and scaled once per sub-tile, before the wait
                [[maybe_unused]] float wv[8];
                if constexpr (WT) {
                    const float4* wp = reinterpret_cast<const float4*>(wts + e_begin + i * kTE + 8 * ((bt & 31) >> 3));
                    const float4 wa = __ldg(wp), wb = __ldg(wp + 1);
                    wv[0] = wa.x; wv[1] = wa.y; wv[2] = wa.z; wv[3] = wa.w; wv[4] = wb.x; wv[5] = wb.y; wv[6] = wb.z; wv[7] = wb.w;
#pragma unroll
                    for (int v = 0; v < 8; v++) wv[v] = wv[v] == w_max ? 1.0f : __fmul_rn(wv[v], w_inv);
                }
                mbar_wait_parked(&raw_full[rs], rph, 200);
                mbar_wait_parked(&op_empty[os], oph ^ 1, 200);
                // K-major B image: byte(k, e) = (k/8)*512 + (e/8)*128 + (k%8)*16 + (e%8)*2      (LBO = 128, SBO = 512)
                uint8_t* g_hi = smem + C::OFF_G + os * C::G_STAGE;
                float dep = 0.0f;
#pragma unroll
                for (int u = 0; u < NIT; u++) {
                    const int it = bt + 96 * u;
                    if (it >= NITEM) break;
                    const int kg = it >> 5, l = it & 31;
                    const int k = kg * 8 + (l & 7), ce = l >> 3;
                    const uint8_t* grow = smem + C::OFF_RAWG + rs * C::RAWG + k * (kTE * 4);
                    const float4 a = *reinterpret_cast<const float4*>(grow + (((2 * ce) ^ (k & 7)) << 4));
                    const float4 b = *reinterpret_cast<const float4*>(grow + (((2 * ce + 1) ^ (k & 7)) << 4));
                    float g[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                    dep += a.x + b.x;
                    if constexpr (WT) {
#pragma unroll
                        for (int v = 0; v < 8; v++) g[v] = __fmul_rn(g[v], wv[v]);
                    }
                    float hi[8], lo[8];
#pragma unroll
                    for (int v = 0; v < 8; v++) {              // gh = 16 * round(64 g) (0 .. 1024), gl = 1024 g - gh, both from the exact product
                        hi[v] = __fsub_rn(__fmaf_rn(g[v], kGammaScale, kGammaMagic), kGammaMagic);
                        lo[v] = __fmaf_rn(g[v], kGammaScale, -hi[v]);
                    }
                    *reinterpret_cast<uint4*>(g_hi + kg * 512 + l * 16) =
                        make_uint4(pack_half2(hi[0], hi[1]), pack_half2(hi[2], hi[3]), pack_half2(hi[4], hi[5]), pack_half2(hi[6], hi[7]));
                    *reinterpret_cast<uint4*>(g_hi + C::G_PART + kg * 512 + l * 16) =
                        make_uint4(pack_half2(lo[0], lo[1]), pack_half2(lo[2], lo[3]), pack_half2(lo[4], lo[5]), pack_half2(lo[6], lo[7]));
                    *reinterpret_cast<uint4*>(g_hi + 2 * C::G_PART + kg * 512 + l * 16) =
                        make_uint4(pack_half2(g[0] * kGammaScale, g[1] * kGammaScale), pack_half2(g[2] * kGammaScale, g[3] * kGammaScale),
                                   pack_half2(g[4] * kGammaScale, g[5] * kGammaScale), pack_half2(g[6] * kGammaScale, g[7] * kGammaScale));
                }
                // The raw tile must BE in registers before the stage goes back to the TMA producer: an mbarrier arrive does
                // not wait for the warp's outstanding shared-memory loads.  The arrive is therefore made data-dependent on
                // every load of this thread (the asm statement consumes the value, so neither the compiler nor the hardware
                // can retire it before the loads have landed).
                __syncwarp();
                if (lane == 0) mbar_arrive_after(&raw_empty[rs], dep);
                else asm volatile("" ::"f"(dep));
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) mbar_arrive(&op_full[os]);
            }
        }
    } else {
        set_regs<C::REG_C, C::REG_LAUNCH>();
        // ===================== consumers: operand build and wgmma, accumulators in registers =====================
        // consumer warpgroup cw (the shuffle shows ptxas that it is warp-uniform, so the branches on the tile index do not
        // make ptxas serialise the wgmma), its first 64-row half hx (of the 2 MT halves) and that half's feature tile mt
        const int cw = __shfl_sync(0xffffffffu, (warp - 4) >> 2, 0);
        const int hx = HPC == 2 ? 2 * cw : part * C::MT + cw;
        const int mt = hx >> 1;
        const int ct = threadIdx.x - 128;                          // consumer thread 0 .. NCT-1
        const int wq = warp & 3, gid = lane >> 2, qd = lane & 3;
        float* racc = reinterpret_cast<float*>(smem + C::OFF_RACC) + ct;     // [32][NCT]: racc[j * NCT]
#pragma unroll
        for (int j = 0; j < 32; j++) racc[j * C::NCT] = 0.0f;
        // this thread's rows hx * 64 + h * 64 + 16 wq + gid + 8 s (slot 2 h + s): shared factor a, factors b[slot] and
        // rounding constants; stage-relative z-tile addresses of its 8 events (pair p at addr ^ (p << 5)): row r at
        // r * 128 (ones block rows at RAWZ + rho * 128), chunk (qd >> 1) ^ (r & 7), byte 8 (qd & 1)
        constexpr int NSLOT = 2 * HPC;
        uint32_t fa, fb[NSLOT];
        float mg[NSLOT];
        {
            const int* om = opmap + hx * 64 + wq * 16 + gid;
            auto addr = [&](int code) {
                const uint32_t row = code >= kRowOne ? (uint32_t)(C::RAWZ / 128 + code - kRowOne) : (uint32_t)code;
                return row * 128 + ((((uint32_t)qd >> 1) ^ (row & 7)) << 4) + ((uint32_t)qd & 1) * 8;
            };
#pragma unroll
            for (int s = 0; s < NSLOT; s++) {
                const int c = om[(s >> 1) * 64 + (s & 1) * 8];
                const int a = c & 255, b = c >> 8;
                if (s == 0) fa = addr(a);
                fb[s] = addr(b);
                mg[s] = a >= kRowOne && b >= kRowOne ? 0.0f : (a >= kRowOne || b >= kRowOne ? magic.lin : magic.prod);
            }
        }
        const uint32_t zs0 = smem_u32(smem + C::OFF_RAWX);
        float ex[HPC][NCL / 2], rm[HPC][NCL / 2];                  // per half of this consumer: exact group, remainder group
#pragma unroll
        for (int h = 0; h < HPC; h++)
#pragma unroll
            for (int j = 0; j < NCL / 2; j++) { ex[h][j] = 0.0f; rm[h][j] = 0.0f; }
        // Accumulator slot q (0 .. 31) of this thread: half q / (NCL / 2), value q % (NCL / 2).  16 at a time (the empty asm
        // keeps ptxas from hoisting all 32 loads): with every accumulator live, 32 loads in flight would not fit the
        // consumers' registers at D = 24.
        auto add_to_racc = [&](float (&acc)[HPC][NCL / 2]) {
#pragma unroll
            for (int c = 0; c < 2; c++) {
#pragma unroll
                for (int j = 0; j < 16; j++) {
                    const int q = 16 * c + j;
                    racc[q * C::NCT] += acc[q / (NCL / 2)][q % (NCL / 2)];
                }
                asm volatile("" ::: "memory");
            }
        };
        uint32_t fh[2][2][4], fl[2][2][4];                          // two A fragment sets: one in flight, one built
        float2 za[4];
        int held = -1;                                             // responsibility stage of the previous sub-tile while its MMAs may run
        // One MMA group: half h of this consumer for sub-tile i, A fragments in (gh, gl).  Two halves per consumer: the
        // group of half 0 of sub-tile i is issued while half 1 of sub-tile i - 1 runs, half 1 of sub-tile i while half 0 runs.
        // One half: the group of sub-tile i runs while sub-tile i + 1 is built.  Either way each group waits (wait_group 1)
        // for the one before it, whose fragment set the next build overwrites.
        auto group = [&](int i, auto hc, uint32_t (&gh)[2][4], uint32_t (&gl)[2][4]) {
            constexpr int h = decltype(hc)::value;
            const int rs = i % kNRAW, rph = (i / kNRAW) & 1;
            const int os = i % kNST, oph = (i / kNST) & 1;
            const uint32_t zst = zs0 + rs * C::RAWX;
            const uint32_t gam = smem_u32(smem + C::OFF_G + os * C::G_STAGE);
            // a chain starts with its first MMA overwriting the accumulators (the drain leaves them as they are)
            const bool new1 = chain_starts(i, mt), new2 = chain2_starts(i, mt);
            if constexpr (h == 0) {
                mbar_wait_parked(&raw_full[rs], rph, 100);
                load_row(zst + fa, za);
            }
            float2 zb0[4], zb1[4];
            load_row(zst + fb[2 * h], zb0);
            load_row(zst + fb[2 * h + 1], zb1);
            build_half(za, zb0, zb1, mg[2 * h], mg[2 * h + 1], gh, gl);
            if constexpr (h == 0) mbar_wait_parked(&op_full[os], oph, 100);
            wgmma_fence();
            issue_half<NCL>(ex[h], rm[h], gh, gl, gam, new1, new2);
            wgmma_commit();
            if constexpr (h == HPC - 1) {
                // The raw stage goes back to the TMA producer only after this warp's loads from it have landed (an mbarrier
                // arrive alone does not wait for them, see the responsibility warps).  The groups of this sub-tile read A
                // fragments computed from every z this thread loaded: the warpgroup-wide wgmma cannot issue before all of
                // them are in registers, and the arrive follows it.
                __syncwarp();
                if (lane == 0) mbar_arrive(&raw_empty[rs]);
            }
            wgmma_wait<1>();
            if constexpr (h == 0) {
                // the previous sub-tile's last group has retired: its responsibility stage is free
                __syncwarp();
                if (lane == 0 && held >= 0) mbar_arrive(&op_empty[held]);
            }
            if constexpr (h == HPC - 1) {
                held = os;
                // drain: exact group at the end of its 128-event chain, remainder group at the end of its longer chain
                // (the second ends only where the first does)
                if (chain_ends(i, mt, nsub)) {
                    wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&op_empty[os]);
                    held = -1;
#if GMM_MSTEP_CUT != 3
                    add_to_racc(ex);
                    if (chain2_ends(i, mt, nsub)) add_to_racc(rm);
#endif
                }
            }
        };
        using H0 = std::integral_constant<int, 0>;
        using H1 = std::integral_constant<int, 1>;
        if constexpr (HPC == 2) {
            for (int i = 0; i < nsub; i++) {
                group(i, H0{}, fh[0], fl[0]);
                group(i, H1{}, fh[1], fl[1]);
            }
        } else {
            // whole pairs, then an odd last sub-tile: a skipped second group inside the loop would give ptxas a path on
            // which set 0 is rebuilt while its group runs, and it would serialise the wgmma (C7513)
            int i = 0;
            for (; i + 1 < nsub; i += 2) {
                group(i, H0{}, fh[0], fl[0]);
                group(i + 1, H0{}, fh[1], fl[1]);
            }
            if (i < nsub) group(i, H0{}, fh[0], fl[0]);
        }
        wgmma_wait<0>();            // (the last sub-tile drained: nothing in flight; without it ptxas waits in every iteration)
#if GMM_MSTEP_CUT == 3
#pragma unroll
        for (int h = 0; h < HPC; h++)
#pragma unroll
            for (int j = 0; j < NCL / 2; j++) ex[h][j] += rm[h][j];
        add_to_racc(ex);
#endif
        // one plain store of this thread's partial sums: [32-cluster block][range][tile][row][32 clusters], the layout
        // mstep_tc_finalize_kernel reduces (the same for both schedules)
        const int nranges = gridDim.x * HPC / 2;
#pragma unroll
        for (int h = 0; h < HPC; h++)
#pragma unroll
            for (int j = 0; j < NCL / 2; j += 2) {
                const int q = h * (NCL / 2) + j;
                const int row = ((hx & 1) + h) * 64 + wq * 16 + gid + 8 * ((j >> 1) & 1);
                const int col = (j >> 2) * 8 + 2 * qd;
                const int ty = blockIdx.y * (NCL / kNCL) + col / kNCL;
                float* dst = scratch + ((((size_t)ty * nranges + range) * C::MT + mt) * 128 + row) * kNCL + col % kNCL;
                *reinterpret_cast<float2*>(dst) = make_float2(racc[q * C::NCT], racc[(q + 1) * C::NCT]);
            }
    }
}

// z = (x - shift) * inv_scale over the SoA event copy, once per data set: the centred/scaled copy the M-step
// tiles are cut from (the E-step converters apply the same two operations to the AoS rows, so both kernels
// see bit-identical z).
__global__ void standardise_soa_kernel(const float* __restrict__ xs, float* __restrict__ zs, size_t pitch, int n, int D,
                                       const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f) {
    const int d = blockIdx.y;
    const float s = shift_f[d], isc = inv_scale_f[d];
    const float* x = xs + (size_t)d * pitch;
    float* z = zs + (size_t)d * pitch;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
        z[e] = __fmul_rn(__fsub_rn(x[e], s), isc);
}

// Reduce the per-CTA FP32 partials in double, undo the operand scaling and write the packed statistics.
// rowmap[row] = (packed statistic index or -1, dimension i, dimension j) of operand row `row` (tc_row_info).
// wscale: the largest weight, which the weighted M-step divided the weights by (1 without weights: no bit changes).
__global__ void __launch_bounds__(256)
mstep_tc_finalize_kernel(const float* __restrict__ scratch, int ncta_x, int MT, int K, int F, const int3* __restrict__ rowmap,
                         const double* __restrict__ scale, double* __restrict__ stats, double wscale) {
    // one block per operand row; thread -> (cluster column, eighth of the CTAs): 128-byte coalesced reads
    constexpr int NQ = 256 / kNCL;
    __shared__ double part[NQ][kNCL];
    const int3 rm = rowmap[blockIdx.x];
    if (rm.x < 0) return;
    const int mt = blockIdx.x / 128, row = blockIdx.x % 128;
    const int col = threadIdx.x & (kNCL - 1), q = threadIdx.x / kNCL;
    double fac = wscale / (double)kGammaScale;
    if (rm.y >= 0) fac *= scale[rm.y];
    if (rm.z >= 0) fac *= scale[rm.z];
    for (int ty = 0; ty * kNCL < K; ty++) {
        double s = 0;
        for (int cx = q; cx < ncta_x; cx += NQ)
            s += (double)scratch[(((size_t)(ty * ncta_x + cx) * MT + mt) * 128 + row) * kNCL + col];
        part[q][col] = s;
        __syncthreads();
        const int k = ty * kNCL + col;
        if (q == 0 && k < K) {
            double t = 0;
#pragma unroll
            for (int u = 0; u < NQ; u++) t += part[u][col];
            stats[(size_t)k * F + rm.x] += t * fac;
        }
        __syncthreads();
    }
}

// ===========================================================================
// E-step (estep1 + estep2 of the reference, gaussian_kernel.cu:383-512) on
// tensor cores.  With Rinv = W^T W (W upper triangular, from the Cholesky
// factor of Rinv) the quadratic form is
//     q_k(x) = || W_k (x - mu_k) ||^2 = || W'_k z + v_k ||^2 ,   z = (x - shift) * inv_scale,
// i.e. ONE GEMM  Y[n][(k,d)] = Z~[n][:] . B[(k,d)][:]  with the constant folded in
// through a ones column, followed by a square-and-sum epilogue, the log-sum-exp
// over the clusters and the log-likelihood reduction.  Operands are FP16 hi/lo
// split (z = zh + zl, W' = Wh + Wl); the products kept are zh Wh, zl Wh, zh Wl and
// 1 v (the lo*lo product is dropped), FP32 accumulation in registers.  The whole
// B operand (all clusters of a pass: 168 KB at K=64, D=24) is RESIDENT in the
// shared memory of one CTA; only the events stream, and they never touch shared
// memory: each thread converts its own rows straight into wgmma A fragments
// (register operand), so one k-step may pair ANY two B chunks (start + LBO).
//
// One persistent CTA per SM, NWG independent warpgroups; each takes 64-event tiles in turn.  Per supergroup of 16 clusters,
// block c of 8 output dimensions and half of the supergroup it issues the k-steps that block needs (m64n64k16, A from
// registers) as one MMA group, and squares and sums the 8 columns of each cluster (a quad of lanes holds them) while the
// next group runs (tc_tile_logits); then the log-sum-exp over the clusters (again within the quad), the responsibilities
// and the log-likelihood.  The other warpgroup's MMAs cover this one's log-sum-exp and stores.
// ===========================================================================

// Block structure.  W is upper triangular, so the 8 output columns d in [8c, 8c+8) of a cluster
// ("block" c) only need the K chunks z_j with j >= c.  Columns are therefore grouped by block:
// one MMA N tile = block c of 16 clusters (N = 128), and block c issues only the k-steps it needs —
// 5 + 4 + 2 = 11 instead of 15 at D = 24.
template <int D> struct ECfg {
    static_assert(D % 8 == 0, "tensor E-step: D must be a multiple of 8");
    static constexpr int CP = D / 8;                          // 8-wide chunks of z / blocks of output columns
    static constexpr int NLO = (CP + 1 + 1) / 2 * 2;          // chunks of the [Wl | v (| pad)] part of the B image
    static constexpr int NCHKB = CP + NLO;                    // B image chunks: Wh_c, then Wl.., v, pad
    static constexpr int GB = 16;                             // clusters per supergroup
    static constexpr int N = GB * 8;                          // MMA N = one block of a supergroup (128 columns)
    static constexpr int MAXSG = 64 / GB;                     // up to 64 clusters resident
    static constexpr int B_BLOCK = NCHKB * N * 16;            // one block of one supergroup
    static constexpr int B_SG = CP * B_BLOCK;
    static constexpr int OFF_B = 0;
    static constexpr int OFF_CK = OFF_B + MAXSG * B_SG;       // float[64] (constant + ln(pi)) * log2(e), then float[64] -0.5 * log2(e) / scale_k^2
    static constexpr int OFF_SH = OFF_CK + 512;               // float[32] shift, float[32] inverse scale
    static constexpr int OFF_BAR = OFF_SH + 256;
    static constexpr int SMEM_BYTES = OFF_BAR + 64;
    static constexpr int NWG = 2;                             // warpgroups per CTA (up to 255 registers each, no spills)
    static constexpr int THREADS = 128 * NWG;
};

// Launch configuration of estep_tc_kernel (score_tc_kernel keeps ECfg's): two MMA warpgroups and two epilogue warpgroups
// per CTA.  An MMA warpgroup writes the base-2 logits of its tile to a slot of a ring in shared memory; epilogue warpgroup
// j takes the tiles of MMA warpgroup j from the ring and does their log-sum-exp, log-likelihood and stores.
//   slot   [64 events][64 clusters] fp32, 256 B per event; the 4-cluster chunk c of event e at chunk c ^ slot_swz(e)
//   stat   [slot][64 events] fp32 subtrahend (the row maximum, or the known log-denominator in base 2), then the scale
//   full / empty  [slot][use parity] mbarriers, 128 arrivals each (the writing MMA warpgroup / the reading epilogue
//                 warpgroup).  Use u of slot s is tile 3 u + s, so successive uses of a slot alternate between the two
//                 warpgroup pairs; with one barrier per use parity each barrier serves one pair only and no waiter can
//                 be two phases behind it (a parity wait on a barrier two phases behind would pass at once).
// D = 8 keeps the fused schedule (estep_fused) and ECfg's configuration.
template <int D> struct EsCfg {
    using E = ECfg<D>;
    static constexpr bool SPLIT = D > 8;
    static constexpr int NMMA = 2;                             // MMA warpgroups, and as many epilogue warpgroups
    static constexpr int THREADS = SPLIT ? 128 * 2 * NMMA : E::THREADS;
    static constexpr int NSLOT = 3;
    static constexpr int SLOT = 64 * 64 * 4;
    static constexpr int OFF_SLOT = (E::SMEM_BYTES + 127) / 128 * 128;
    static constexpr int OFF_STAT = OFF_SLOT + NSLOT * SLOT;
    static constexpr int OFF_EBAR = OFF_STAT + NSLOT * 2 * 64 * 4;
    static constexpr int SMEM_BYTES = SPLIT ? OFF_EBAR + 4 * NSLOT * 8 : E::SMEM_BYTES;
    // register pools (setmaxnreg redistributes the launch allocation of REG_LAUNCH per thread, see MCfg)
    static constexpr int REG_LAUNCH = 65536 / (128 * 2 * NMMA) / 8 * 8;
    static constexpr int REG_MMA = 184;
    static constexpr int REG_EPI = 72;
    static_assert(128 * NMMA * (REG_MMA + REG_EPI) <= 128 * 2 * NMMA * REG_LAUNCH, "register pools");
    static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

// Physical chunk offset of event e in a logit slot.  Conflict-free (one wavefront per 8 lanes of a 16-byte access) for
// the three access patterns: the MMA lanes' writes (a quarter warp: events e, e + 1, every chunk of a supergroup), the
// epilogue's row reads (4 consecutive events, chunks c, c ^ 1) and its block reads (one chunk, events 4a + j, 8 values of a).
__device__ __forceinline__ uint32_t slot_swz(int e) { return (uint32_t)(((e & 1) << 2 | (e & 2)) ^ ((e >> 2) & 7)); }

__device__ __forceinline__ void sts_f4(uint32_t addr, float a, float b, float c, float d) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
// named barrier 1 + j of epilogue warpgroup j alone (barrier 0 is __syncthreads)
__device__ __forceinline__ void epi_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Timing variants of the E-step for scripts/prof_estep.py (`make variant DEFS=-DGMM_ESTEP_CUT=n`); the default build is 0.
//   1  MMA only: the accumulators feed one sum per block, no squares, log-sum-exp, exp, log or stores (results are wrong)
//   2  no stores: the full epilogue, but the responsibilities are not written
#ifndef GMM_ESTEP_CUT
#define GMM_ESTEP_CUT 0
#endif

// ---- pieces shared by estep_tc_kernel and score_tc_kernel (same operand path, different epilogues) ----------------
// Shared-memory staging of one pass: constants, shift / inverse scale, and the resident B image (one TMA bulk copy per
// block, completion on b_full).  Followed by a __syncthreads inside; the caller waits on b_full before the first MMA.
template <int D>
__device__ __forceinline__ void tc_stage_operand(uint8_t* smem, const uint8_t* __restrict__ b_img, const float* __restrict__ ck,
                                                 const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f, int NSG) {
    using C = ECfg<D>;
    uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
    float* ck_s = reinterpret_cast<float*>(smem + C::OFF_CK);
    float* sh_s = reinterpret_cast<float*>(smem + C::OFF_SH);
    if (threadIdx.x == 0) { mbar_init(b_full, 1); fence_mbar_init(); }
    // base-2 logits in the epilogue: l2 = ck * log2(e) + (-0.5 * log2(e) / scale_k^2) * |scale_k * y|^2   (the per-cluster
    // power-of-two scale_k keeps the FP16 whitening factors in range whatever the cluster's width, see bimg_cluster)
    if (threadIdx.x < 64) { ck_s[threadIdx.x] = ck[threadIdx.x] * 1.4426950408889634f; ck_s[64 + threadIdx.x] = ck[64 + threadIdx.x]; }
    if (threadIdx.x < D) { sh_s[threadIdx.x] = shift_f[threadIdx.x]; sh_s[32 + threadIdx.x] = inv_scale_f[threadIdx.x]; }
    __syncthreads();
    if (threadIdx.x == 0) {                    // resident B operand: one TMA bulk copy per block
        mbar_arrive_expect_tx(b_full, (uint32_t)NSG * C::B_SG);
        for (int g = 0; g < NSG * C::CP; g++) tma_load_1d(smem + C::OFF_B + g * C::B_BLOCK, b_img + (size_t)g * C::B_BLOCK, C::B_BLOCK, b_full);
    }
}

// Standardise the two rows a thread holds and split them into FP16 hi / lo A fragments ([chunk][row]).
template <int D>
__device__ __forceinline__ void tc_split_rows(const float2 (&xa)[D / 8], const float2 (&xb)[D / 8], const float* sh_s, const float* isc_s,
                                              int qd, uint32_t (&zh)[D / 8][2], uint32_t (&zl)[D / 8][2]) {
#pragma unroll
    for (int j = 0; j < D / 8; j++) {
        const float s0 = sh_s[8 * j + 2 * qd], s1 = sh_s[8 * j + 2 * qd + 1];
        const float i0 = isc_s[8 * j + 2 * qd], i1 = isc_s[8 * j + 2 * qd + 1];
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const float2 x = r ? xb[j] : xa[j];
            const float z0 = __fmul_rn(__fsub_rn(x.x, s0), i0), z1 = __fmul_rn(__fsub_rn(x.y, s1), i1);
            const __half2 h = __floats2half2_rn(z0, z1);
            const float2 f = __half22float2(h);
            zh[j][r] = *reinterpret_cast<const uint32_t*>(&h);
            zl[j][r] = pack_half2(z0 - f.x, z1 - f.y);
        }
    }
}

// One MMA group of a tile: half h (clusters 8h .. 8h+7 of the supergroup whose B image starts at bsg, N = 64) of block c,
// i.e. the k-steps that block needs (m64n64k16, A from registers), into a 32-register accumulator.  The first k-step
// overwrites it (scale-d = 0).  The caller commits.
template <int D>
__device__ __forceinline__ void tc_issue_group(float (&acc)[32], const uint32_t (&zh)[D / 8][2], const uint32_t (&zl)[D / 8][2],
                                               uint32_t bsg, int c, int h, uint32_t ones) {
    using C = ECfg<D>;
    constexpr int CP = C::CP;
    constexpr uint32_t CH = C::N * 16;                        // bytes per B chunk (128 rows of 16 B)
    const uint32_t bb = bsg + (uint32_t)c * C::B_BLOCK + (uint32_t)h * (CH / 2);
    wgmma_fence();
#pragma unroll
    for (int j = c; j < CP; j++)                              // (Wh_j, Wl_j) x (zh_j, zh_j)
        wgmma_m64n64k16_rs(acc, zh[j][0], zh[j][1], zh[j][0], zh[j][1], make_smem_desc(bb + j * CH, CP * CH, 128), j > c);
    // (Wh_j) x (zl_j) for j >= c, then v x ones, two at a time; a lone v step pairs with a zero A chunk
#pragma unroll
    for (int p = c; p < CP + 1; p += 2) {
        const int x = p, y = p + 1;                           // list items: j < CP -> Wh_j x zl_j, j == CP -> v x ones
        if (y <= CP) {
            const uint32_t yc = y < CP ? (uint32_t)y : 2u * CP;
            const uint32_t a2 = y < CP ? zl[y < CP ? y : 0][0] : ones, a3 = y < CP ? zl[y < CP ? y : 0][1] : ones;
            wgmma_m64n64k16_rs(acc, zl[x][0], zl[x][1], a2, a3, make_smem_desc(bb + x * CH, (yc - x) * CH, 128), true);
        } else {                                              // x == CP: v alone, paired with chunk c under a zero A chunk
            wgmma_m64n64k16_rs(acc, 0u, 0u, ones, ones, make_smem_desc(bb + c * CH, (2 * CP - c) * CH, 128), true);
        }
    }
}

// The base-2 logits of one 64-event tile against the resident clusters of the pass: per supergroup of 16 clusters, block
// c of 8 output dimensions and half h of the supergroup's clusters the k-steps that block needs (one MMA group), the
// squares summed over the 8 columns of each cluster with a quad transpose.  lg[sg][u]: cluster sg * 16 + 8 (qd & 1) +
// 4 (qd >> 1) + (u >> 1), row u & 1 (-inf for supergroups >= NSG).
// Software pipeline: the groups (sg, c, h) form one sequence over a ring of two accumulators (group (sg, c, h) in acc[h]);
// group i + 1 is issued and committed before group i is waited for and squared, so this warpgroup always has MMAs queued
// while it squares and transposes; only the tile's last group is waited for with nothing behind it.  No group stays in
// flight across tiles: the register A operand zh / zl of the next tile could not be written while this tile's last group
// still reads it, and ptxas serialises every wgmma when a pending group is carried around the tile loop.
// NSG (resident supergroups of the pass) is a template parameter: with a wgmma issue or a wait<1> under a run-time branch
// on it, ptxas serialises every wgmma of the kernel (C7514).
template <int D, int NSG>
__device__ __forceinline__ void tc_tile_logits(const uint32_t (&zh)[D / 8][2], const uint32_t (&zl)[D / 8][2], uint32_t bsm,
                                               const float* ck_s, int qd, uint32_t ones, float (&lg)[ECfg<D>::MAXSG][8]) {
    using C = ECfg<D>;
    constexpr int CP = C::CP;
    float acc[2][32];
    tc_issue_group<D>(acc[0], zh, zl, bsm, 0, 0, ones);
    wgmma_commit();
#pragma unroll
    for (int sg = 0; sg < C::MAXSG; sg++) {
        if (sg >= NSG) {
#pragma unroll
            for (int u = 0; u < 8; u++) lg[sg][u] = -INFINITY;
            continue;
        }
        const uint32_t bsg = bsm + (uint32_t)sg * C::B_SG;
        float sq[32];                                      // sums of squares: [cluster 0..15][row]
#pragma unroll
        for (int u = 0; u < 32; u++) sq[u] = 0.f;
#pragma unroll
        for (int c = 0; c < CP; c++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                // queue the next group of the sequence, then wait for this one (all conditions are compile-time)
                if (sg + 1 == NSG && c + 1 == CP && h == 1) {
                    wgmma_wait<0>();
                } else {
                    if (h == 0) tc_issue_group<D>(acc[1], zh, zl, bsg, c, 1, ones);
                    else if (c + 1 < CP) tc_issue_group<D>(acc[0], zh, zl, bsg, c + 1, 0, ones);
                    else tc_issue_group<D>(acc[0], zh, zl, bsg + C::B_SG, 0, 0, ones);
                    wgmma_commit();
                    wgmma_wait<1>();
                }
                wgmma_pin(acc[h]);
                const float(&a)[32] = acc[h];
#if GMM_ESTEP_CUT == 1
                sq[0] += a[0];
#else
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    float& s0 = sq[16 * h + 2 * i];
                    float& s1 = sq[16 * h + 2 * i + 1];
                    s0 = fmaf(a[4 * i], a[4 * i], fmaf(a[4 * i + 1], a[4 * i + 1], s0));
                    s1 = fmaf(a[4 * i + 2], a[4 * i + 2], fmaf(a[4 * i + 3], a[4 * i + 3], s1));
                }
#endif
            }
        }
#if GMM_ESTEP_CUT == 1
        for (int u = 0; u < 8; u++) lg[sg][u] = sq[0];
        continue;
#endif
        // sum over the quad (the 8 columns of a cluster are spread over its 4 lanes), transposing as it goes:
        // lane qd ends with clusters cb .. cb+3 of the supergroup, cb = 8 (qd & 1) + 4 (qd >> 1), both rows
        float w[16];
        const bool b1 = qd & 1, b2 = (qd >> 1) & 1;
#pragma unroll
        for (int u = 0; u < 16; u++) {
            const float send = b1 ? sq[u] : sq[16 + u], keep = b1 ? sq[16 + u] : sq[u];
            w[u] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const float send = b2 ? w[u] : w[8 + u], keep = b2 ? w[8 + u] : w[u];
            const float qv = keep + __shfl_xor_sync(0xffffffffu, send, 2);
            const int k = sg * C::GB + 8 * (qd & 1) + 4 * (qd >> 1) + (u >> 1);
            lg[sg][u] = fmaf(ck_s[64 + k], qv, ck_s[k]);
        }
    }
}

// The MMA side of one 64-event tile of the E-step: the groups, squares and quad transpose of tc_tile_logits in the same
// order, over a ring of two accumulators (group g + 1 is issued and committed before group g is waited for and squared; a
// third accumulator fits the register pool without spills but measured slower), and each supergroup's 8 base-2 logits per thread written to the logit slot at `slot` (two 16-byte
// stores: 4 clusters of one event each) instead of being kept in registers.  Supergroups >= NSG are not written: the
// epilogue does not read them.
template <int D, int NSG>
__device__ __forceinline__ void estep_tile_logits(const uint32_t (&zh)[D / 8][2], const uint32_t (&zl)[D / 8][2], uint32_t bsm,
                                                  const float* ck_s, int qd, uint32_t ones, uint32_t slot, int r0, float& cut_sum) {
    using C = ECfg<D>;
    constexpr int CP = C::CP, NG = NSG * CP * 2;
    float acc[2][32];
    tc_issue_group<D>(acc[0], zh, zl, bsm, 0, 0, ones);
    wgmma_commit();
    const uint32_t cq = 2 * (qd & 1) + (qd >> 1);             // this lane's chunk of 4 clusters within a supergroup
    const uint32_t row0 = slot + (uint32_t)r0 * 256, row1 = row0 + 8 * 256;
    const uint32_t sw0 = slot_swz(r0), sw1 = slot_swz(r0 + 8);
    float sq[32];                                             // sums of squares of a supergroup: [cluster 0..15][row]
#pragma unroll
    for (int g = 0; g < NG; g++) {
        const int sg = g / (2 * CP), c = (g / 2) % CP, h = g & 1;
        if (c == 0 && h == 0) {
#pragma unroll
            for (int u = 0; u < 32; u++) sq[u] = 0.f;
        }
        // queue group g + 1, then wait for group g (all conditions are compile-time)
        if (g + 1 < NG) {
            const int gn = g + 1;
            tc_issue_group<D>(acc[gn & 1], zh, zl, bsm + (uint32_t)(gn / (2 * CP)) * C::B_SG, (gn / 2) % CP, gn & 1, ones);
            wgmma_commit();
            wgmma_wait<1>();
        } else {
            wgmma_wait<0>();
        }
        wgmma_pin(acc[g & 1]);
        const float(&a)[32] = acc[g & 1];
#if GMM_ESTEP_CUT == 1
        cut_sum += a[0];
#else
#pragma unroll
        for (int i = 0; i < 8; i++) {
            float& s0 = sq[16 * h + 2 * i];
            float& s1 = sq[16 * h + 2 * i + 1];
            s0 = fmaf(a[4 * i], a[4 * i], fmaf(a[4 * i + 1], a[4 * i + 1], s0));
            s1 = fmaf(a[4 * i + 2], a[4 * i + 2], fmaf(a[4 * i + 3], a[4 * i + 3], s1));
        }
        if (c == CP - 1 && h == 1) {
            // sum over the quad, transposing as it goes (tc_tile_logits): lane qd ends with clusters cb .. cb+3 of the
            // supergroup, cb = 8 (qd & 1) + 4 (qd >> 1) = 4 cq, both rows
            float w[16];
            const bool b1 = qd & 1, b2 = (qd >> 1) & 1;
#pragma unroll
            for (int u = 0; u < 16; u++) {
                const float send = b1 ? sq[u] : sq[16 + u], keep = b1 ? sq[16 + u] : sq[u];
                w[u] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
            }
            float l[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const float send = b2 ? w[u] : w[8 + u], keep = b2 ? w[8 + u] : w[u];
                const float qv = keep + __shfl_xor_sync(0xffffffffu, send, 2);
                const int k = sg * C::GB + 8 * (qd & 1) + 4 * (qd >> 1) + (u >> 1);
                l[u] = fmaf(ck_s[64 + k], qv, ck_s[k]);
            }
            const uint32_t ch = 4 * (uint32_t)sg + cq;
            sts_f4(row0 + ((ch ^ sw0) << 4), l[0], l[2], l[4], l[6]);
            sts_f4(row1 + ((ch ^ sw1) << 4), l[1], l[3], l[5], l[7]);
        }
#endif
    }
}

// The fused schedule (D = 8): two warpgroups, each doing the MMAs, log-sum-exp and stores of its own tiles, with
// ECfg's launch configuration.  Called by estep_tc_kernel; see there for the modes.
template <int D, int NSG, bool WT>
__device__ __forceinline__ void estep_fused(const float* __restrict__ x_aos, const uint8_t* __restrict__ b_img, const float* __restrict__ ck,
                const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f, float* __restrict__ memb,
                size_t pitch, int n, int K, double* __restrict__ ll_out, int mode, const float* den_in, float* den_out,
                const float* __restrict__ wts) {
    // K / NSG (= ceil(K / 16)) / b_img / ck / memb describe ONE pass of at most 64 clusters.  More than 64 clusters take 2P - 1 launches
    // for P passes, and every responsibility is written exactly once:
    //   mode 1 (passes 0 .. P-2)  log-denominator only: den_out[e] = ln(sum_k exp(logit)) (+ den_in[e] in log space), no stores
    //   mode 2 (pass P-1)         its own log-sum-exp joined with den_in[e] (all other passes): final responsibilities of this
    //                             pass, den_out[e] = the event's total log-denominator, log-likelihood
    //   mode 3 (passes 0 .. P-2)  responsibilities against the known total den_in[e]: no log-sum-exp
    //   mode 0                    single pass (K <= 64)
    // WT (gmm_set_weights): the log-likelihood adds wts[e] * denominator; the responsibilities do not depend on the weights.
    using C = ECfg<D>;
    constexpr int CP = C::CP;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
    float* ck_s = reinterpret_cast<float*>(smem + C::OFF_CK);          // [64] additive logit constants, [64] multipliers
    float* sh_s = reinterpret_cast<float*>(smem + C::OFF_SH);          // [32] shift, [32] inverse scale
    float* isc_s = sh_s + 32;

    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int gid = lane >> 2, qd = lane & 3;
    const int ntiles = (n + 63) / 64;

    tc_stage_operand<D>(smem, b_img, ck, shift_f, inv_scale_f, NSG);

    // rows r0 = 16 warp + gid and r1 = r0 + 8 of each 64-event tile; K positions 2 qd, 2 qd + 1 of every 8-wide chunk
    const int r0 = warp * 16 + gid;
    float2 xa[CP], xb[CP];                     // raw coordinates of the two rows (prefetched one tile ahead)
    auto load_rows = [&](int t) {
        const long long e0 = (long long)t * 64 + r0, e1 = e0 + 8;
#pragma unroll
        for (int j = 0; j < CP; j++) {
            xa[j] = e0 < n ? __ldg(reinterpret_cast<const float2*>(x_aos + (size_t)e0 * D + 8 * j + 2 * qd)) : make_float2(0.f, 0.f);
            xb[j] = e1 < n ? __ldg(reinterpret_cast<const float2*>(x_aos + (size_t)e1 * D + 8 * j + 2 * qd)) : make_float2(0.f, 0.f);
        }
    };
    const int stride = (int)gridDim.x * C::NWG;
    int t = (int)blockIdx.x * C::NWG + wg;
    if (t < ntiles) load_rows(t);
    const uint32_t ones = qd == 0 ? 0x3C003C00u : 0u;         // chunk {1, 1, 0 ...}: K elements 0 and 1 are held by qd == 0
    const uint32_t bsm = smem_u32(smem + C::OFF_B);
    double ll_acc = 0.0;
    constexpr float kLn2 = 0.6931471805599453f;
    mbar_wait(b_full, 0);

    for (; t < ntiles; t += stride) {
        uint32_t zh[CP][2], zl[CP][2];                         // [chunk][row]: FP16 pairs, hi and lo parts
        tc_split_rows<D>(xa, xb, sh_s, isc_s, qd, zh, zl);
        const long long e0 = (long long)t * 64 + r0, e1 = e0 + 8;
        if (t + stride < ntiles) load_rows(t + stride);

        float lg[C::MAXSG][8];                                 // base-2 logits: [supergroup][4 clusters x 2 rows]
        tc_tile_logits<D, NSG>(zh, zl, bsm, ck_s, qd, ones, lg);
#if GMM_ESTEP_CUT == 1
        for (int sg = 0; sg < C::MAXSG; sg++) ll_acc += (double)lg[sg][0];
        continue;
#endif
        // log-sum-exp over the clusters (estep2, gaussian_kernel.cu:481-503), per row: this lane's 16 logits, then the quad.
        // The maximum starts at -FLT_MAX: in a pass whose clusters all have pi = 0 (logits -inf) every term is then
        // ex2(-inf) = 0 rather than NaN, S = 0 and the pass's log-denominator -inf; any finite logit sets it as before
        float mx[2] = {-FLT_MAX, -FLT_MAX};
#pragma unroll
        for (int sg = 0; sg < C::MAXSG; sg++)
#pragma unroll
            for (int u = 0; u < 8; u++) mx[u & 1] = fmaxf(mx[u & 1], lg[sg][u]);
#pragma unroll
        for (int r = 0; r < 2; r++) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        }
        float scale[2] = {1.f, 1.f};
        const long long er[2] = {e0, e1};
        if (mode == 3) {
            // the event's total log-denominator is known: gamma = 2^(l2 - denom * log2 e)
            float d2[2];
#pragma unroll
            for (int r = 0; r < 2; r++) d2[r] = er[r] < n ? den_in[er[r]] * 1.4426950408889634f : 0.f;
#pragma unroll
            for (int sg = 0; sg < C::MAXSG; sg++)
#pragma unroll
                for (int u = 0; u < 8; u++) lg[sg][u] = ex2_approx(lg[sg][u] - d2[u & 1]);
        } else {
            float sm[2] = {0.f, 0.f};
#pragma unroll
            for (int sg = 0; sg < C::MAXSG; sg++)
#pragma unroll
                for (int u = 0; u < 8; u++) { lg[sg][u] = ex2_approx(lg[sg][u] - mx[u & 1]); sm[u & 1] += lg[sg][u]; }
            float dx[2];
#pragma unroll
            for (int r = 0; r < 2; r++) {
                sm[r] += __shfl_xor_sync(0xffffffffu, sm[r], 1);
                sm[r] += __shfl_xor_sync(0xffffffffu, sm[r], 2);
                // den_in may alias den_out (running log-denominator updated in place): every lane reads before any writes
                dx[r] = (mode != 0 && den_in != nullptr && er[r] < n) ? den_in[er[r]] : 0.f;
            }
            __syncwarp();
#pragma unroll
            for (int r = 0; r < 2; r++) {
                float denom = fmaf(mx[r], kLn2, logf(sm[r]));      // :490-494, back in natural units
                scale[r] = 1.0f / sm[r];                            // exp(l - denom) = 2^(l2 - M) / S
                if (mode != 0 && er[r] < n) {
                    if (den_in != nullptr) {                        // join with the other passes' log-denominator
                        // floored at -FLT_MAX: two -inf operands (passes without a finite logit) join to -inf, not NaN
                        const float g = fmaxf(fmaxf(denom, dx[r]), -FLT_MAX);
                        const float tot = g + logf(__expf(denom - g) + __expf(dx[r] - g));
                        // S = 0 (no finite logit in this pass): its terms are all 0 and so are its responsibilities
                        scale[r] = sm[r] == 0.f ? 0.f : scale[r] * __expf(denom - tot);
                        denom = tot;
                    }
                    if (qd == 0) den_out[er[r]] = denom;
                }
                if constexpr (WT) {
                    if (qd == 0 && er[r] < n && (mode == 0 || mode == 2)) ll_acc += (double)wts[er[r]] * (double)denom;
                } else {
                    if (qd == 0 && er[r] < n && (mode == 0 || mode == 2)) ll_acc += (double)denom;
                }
            }
        }
        if (mode != 1 && GMM_ESTEP_CUT != 2) {
            // Rows [K, 8*ceil(K/8)) are written too (zeros of the padding clusters): the buffer is allocated in
            // multiples of 8 rows.
#pragma unroll
            for (int sg = 0; sg < C::MAXSG; sg++) {
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const int k = sg * C::GB + 8 * (qd & 1) + 4 * (qd >> 1) + (u >> 1);
                    const long long e = er[u & 1];
                    if (sg < NSG && (k & ~7) < K && e < n) memb[(size_t)k * pitch + e] = lg[sg][u] * scale[u & 1];   // :498-501
                }
            }
        }
    }
    if (mode == 0 || mode == 2) {
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 16);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 8);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 4);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 2);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 1);
        if (lane == 0) atomicAdd(ll_out, ll_acc);
    }
}

template <int D, int NSG, bool WT = false>
__global__ void __launch_bounds__(EsCfg<D>::THREADS, 1)
estep_tc_kernel(const float* __restrict__ x_aos, const uint8_t* __restrict__ b_img, const float* __restrict__ ck,
                const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f, float* __restrict__ memb,
                size_t pitch, int n, int K, double* __restrict__ ll_out, int mode, const float* den_in, float* den_out,
                const float* __restrict__ wts) {
    // K / NSG (= ceil(K / 16)) / b_img / ck / memb describe ONE pass of at most 64 clusters.  More than 64 clusters take 2P - 1 launches
    // for P passes, and every responsibility is written exactly once:
    //   mode 1 (passes 0 .. P-2)  log-denominator only: den_out[e] = ln(sum_k exp(logit)) (+ den_in[e] in log space), no stores
    //   mode 2 (pass P-1)         its own log-sum-exp joined with den_in[e] (all other passes): final responsibilities of this
    //                             pass, den_out[e] = the event's total log-denominator, log-likelihood
    //   mode 3 (passes 0 .. P-2)  responsibilities against the known total den_in[e]: no log-sum-exp
    //   mode 0                    single pass (K <= 64)
    // WT (gmm_set_weights): the log-likelihood adds wts[e] * denominator; the responsibilities do not depend on the weights.
    if constexpr (!EsCfg<D>::SPLIT) {
        estep_fused<D, NSG, WT>(x_aos, b_img, ck, shift_f, inv_scale_f, memb, pitch, n, K, ll_out, mode, den_in, den_out, wts);
        return;
    } else {
    // The CTA's tile i (i = 0, 1, ...) is tile blockIdx.x * NMMA + i % NMMA + (i / NMMA) * stride of the grid; MMA
    // warpgroup i % NMMA writes its logits to slot i % NSLOT, and epilogue warpgroup i % NMMA reads them from there.
    using E = ECfg<D>;
    using C = EsCfg<D>;
    constexpr int CP = E::CP;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + E::OFF_BAR);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::OFF_EBAR);   // [NSLOT][2] logits written
    uint64_t* empty = full + 2 * C::NSLOT;                              // [NSLOT][2] logits read
    const float* ck_s = reinterpret_cast<const float*>(smem + E::OFF_CK);   // [64] additive logit constants, [64] multipliers
    const float* sh_s = reinterpret_cast<const float*>(smem + E::OFF_SH);   // [32] shift, [32] inverse scale
    const float* isc_s = sh_s + 32;
    const uint32_t slots = smem_u32(smem + C::OFF_SLOT);

    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int ntiles = (n + 63) / 64;
    const int stride = (int)gridDim.x * C::NMMA;
    if (threadIdx.x == 0) {
        for (int b = 0; b < 2 * C::NSLOT; b++) { mbar_init(&full[b], 128); mbar_init(&empty[b], 128); }
    }
    tc_stage_operand<D>(smem, b_img, ck, shift_f, inv_scale_f, NSG);   // fences the barrier inits, then __syncthreads

    if (wg < C::NMMA) {
        // ---- MMA warpgroup: logits of tiles wg, wg + NMMA, ... of the CTA ----
        set_regs<C::REG_MMA, C::REG_LAUNCH>();
        const int gid = lane >> 2, qd = lane & 3;
        // rows r0 = 16 warp + gid and r1 = r0 + 8 of each 64-event tile; K positions 2 qd, 2 qd + 1 of every 8-wide chunk
        const int r0 = warp * 16 + gid;
        float2 xa[CP], xb[CP];                     // raw coordinates of the two rows (prefetched one tile ahead)
        auto load_rows = [&](int t) {
            const long long e0 = (long long)t * 64 + r0, e1 = e0 + 8;
#pragma unroll
            for (int j = 0; j < CP; j++) {
                xa[j] = e0 < n ? __ldg(reinterpret_cast<const float2*>(x_aos + (size_t)e0 * D + 8 * j + 2 * qd)) : make_float2(0.f, 0.f);
                xb[j] = e1 < n ? __ldg(reinterpret_cast<const float2*>(x_aos + (size_t)e1 * D + 8 * j + 2 * qd)) : make_float2(0.f, 0.f);
            }
        };
        int t = (int)blockIdx.x * C::NMMA + wg;
        if (t < ntiles) load_rows(t);
        const uint32_t ones = qd == 0 ? 0x3C003C00u : 0u;         // chunk {1, 1, 0 ...}: K elements 0 and 1 are held by qd == 0
        const uint32_t bsm = smem_u32(smem + E::OFF_B);
        float cut_sum = 0.f;
        mbar_wait(b_full, 0);
        for (int i = wg; t < ntiles; t += stride, i += C::NMMA) {
            uint32_t zh[CP][2], zl[CP][2];                         // [chunk][row]: FP16 pairs, hi and lo parts
            tc_split_rows<D>(xa, xb, sh_s, isc_s, qd, zh, zl);
            if (t + stride < ntiles) load_rows(t + stride);
            const int s = i % C::NSLOT, u = i / C::NSLOT;           // use u of slot s
#if GMM_ESTEP_CUT != 1
            if (u > 0) mbar_wait(&empty[2 * s + ((u - 1) & 1)], ((u - 1) >> 1) & 1);   // use u - 1 read
#endif
            estep_tile_logits<D, NSG>(zh, zl, bsm, ck_s, qd, ones, slots + (uint32_t)s * C::SLOT, r0, cut_sum);
#if GMM_ESTEP_CUT != 1
            mbar_arrive(&full[2 * s + (u & 1)]);
#endif
        }
        if (GMM_ESTEP_CUT == 1 && cut_sum == -1.f) atomicAdd(ll_out, 0.0);   // keeps the variant's MMAs alive
        return;
    }

    // ---- epilogue warpgroup ew: the tiles of MMA warpgroup ew ----
    set_regs<C::REG_EPI, C::REG_LAUNCH>();
    if (GMM_ESTEP_CUT == 1) return;
    const int ew = wg - C::NMMA, et = threadIdx.x & 127;
    // log-sum-exp: two threads per event (ev = et / 2); thread hh holds the P sums of lanes qd = 2 hh and 2 hh + 1 of the
    // MMA quad, i.e. the chunks 4 sg + hh and 4 sg + 2 + hh of every supergroup
    const int ev = et >> 1, hh = et & 1;
    const uint32_t evrow = (uint32_t)ev * 256, evswz = slot_swz(ev);
    float* stat = reinterpret_cast<float*>(smem + C::OFF_STAT);          // [NSLOT][subtrahend 64 | scale 64]
    const uint32_t stat_u = smem_u32(stat);
    double ll_acc = 0.0;
    constexpr float kLn2 = 0.6931471805599453f, kLog2e = 1.4426950408889634f;
    for (int i = ew;; i += C::NMMA) {
        const int t = (int)blockIdx.x * C::NMMA + i % C::NMMA + (i / C::NMMA) * stride;
        if (t >= ntiles) break;
        const int s = i % C::NSLOT;
        const uint32_t slot = slots + (uint32_t)s * C::SLOT;
        const int u = i / C::NSLOT, sb2 = 2 * s + (u & 1);
        mbar_wait(&full[sb2], (u >> 1) & 1);
        const long long e = (long long)t * 64 + ev;
        float sub, scl = 1.f, dep = 0.f;
        if (mode == 3) {
            // the event's total log-denominator is known: gamma = 2^(l2 - denom * log2 e)
            sub = e < n ? den_in[e] * kLog2e : 0.f;
        } else {
            // log-sum-exp over the clusters (estep2, gaussian_kernel.cu:481-503); the maximum starts at -FLT_MAX, so that a
            // pass without a finite logit (every pi 0) has terms ex2(-inf) = 0, S = 0 and a log-denominator of -inf
            float mx = -FLT_MAX;
#pragma unroll
            for (int sg = 0; sg < NSG; sg++)
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const float4 v = lds_f4(slot + evrow + (((uint32_t)(4 * sg + 2 * j + hh) ^ evswz) << 4));
                    mx = fmaxf(fmaxf(mx, v.x), fmaxf(fmaxf(v.y, v.z), v.w));
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            // S = (P0 + P1) + (P2 + P3), each P_qd = 0 + its 16 terms in (supergroup, cluster) order: the sums of the
            // MMA quad's lanes and of its two shuffle steps, bit for bit
            float p0 = 0.f, p1 = 0.f;
#pragma unroll
            for (int sg = 0; sg < NSG; sg++) {
                const float4 v0 = lds_f4(slot + evrow + (((uint32_t)(4 * sg + hh) ^ evswz) << 4));
                const float4 v1 = lds_f4(slot + evrow + (((uint32_t)(4 * sg + 2 + hh) ^ evswz) << 4));
                p0 += ex2_approx(v0.x - mx); p0 += ex2_approx(v0.y - mx); p0 += ex2_approx(v0.z - mx); p0 += ex2_approx(v0.w - mx);
                p1 += ex2_approx(v1.x - mx); p1 += ex2_approx(v1.y - mx); p1 += ex2_approx(v1.z - mx); p1 += ex2_approx(v1.w - mx);
            }
            const float a = p0 + p1;
            const float S = a + __shfl_xor_sync(0xffffffffu, a, 1);
            sub = mx;
            dep = S;
            if (hh == 0) {
                float denom = fmaf(mx, kLn2, logf(S));              // :490-494, back in natural units
                scl = 1.0f / S;                                     // exp(l - denom) = 2^(l2 - M) / S
                if (mode != 0 && e < n) {
                    if (den_in != nullptr) {                        // join with the other passes' log-denominator
                        const float dx = den_in[e];                 // den_in may alias den_out: read before the write
                        const float g = fmaxf(fmaxf(denom, dx), -FLT_MAX);   // two -inf operands join to -inf
                        const float tot = g + logf(__expf(denom - g) + __expf(dx - g));
                        scl = S == 0.f ? 0.f : scl * __expf(denom - tot);   // S = 0: every term of the pass is 0
                        denom = tot;
                    }
                    den_out[e] = denom;
                }
                if constexpr (WT) {
                    if (e < n && (mode == 0 || mode == 2)) ll_acc += (double)wts[e] * (double)denom;
                } else {
                    if (e < n && (mode == 0 || mode == 2)) ll_acc += (double)denom;
                }
            }
        }
        if (mode == 1 || GMM_ESTEP_CUT == 2) {
            mbar_arrive_after(&empty[sb2], dep);
            continue;
        }
        if (hh == 0) { stat[s * 128 + ev] = sub; stat[s * 128 + 64 + ev] = scl; }
        epi_bar(1 + ew);
        // responsibilities (:498-501) in blocks of 4 events x 4 clusters: lanes 16 b .. 16 b + 15 of a warp hold the 64
        // events of one chunk, so each 16-byte store instruction writes 256 contiguous bytes of each of two cluster rows.
        // Rows [K, 8*ceil(K/8)) are written too (zeros of the padding clusters): the buffer is allocated in multiples of 8 rows.
#pragma unroll 1
        for (int j = 0; j < 2; j++) {
            const int b = et + 128 * j, c = b >> 4, a = b & 15;
            if (c >= 4 * NSG || (4 * c & ~7) >= K) continue;
            float4 v[4];
#pragma unroll
            for (int m = 0; m < 4; m++) v[m] = lds_f4(slot + (uint32_t)(4 * a + m) * 256 + (((uint32_t)c ^ slot_swz(4 * a + m)) << 4));
            const float4 sb = lds_f4(stat_u + (uint32_t)s * 512 + 16 * a), sc = lds_f4(stat_u + (uint32_t)s * 512 + 256 + 16 * a);
            dep += (v[0].x + v[1].x) + (v[2].x + v[3].x);
            const long long e0 = (long long)t * 64 + 4 * a;
            float* dst = memb + (size_t)(4 * c) * pitch + e0;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const float l0 = q == 0 ? v[0].x : q == 1 ? v[0].y : q == 2 ? v[0].z : v[0].w;
                const float l1 = q == 0 ? v[1].x : q == 1 ? v[1].y : q == 2 ? v[1].z : v[1].w;
                const float l2 = q == 0 ? v[2].x : q == 1 ? v[2].y : q == 2 ? v[2].z : v[2].w;
                const float l3 = q == 0 ? v[3].x : q == 1 ? v[3].y : q == 2 ? v[3].z : v[3].w;
                const float4 gm = make_float4(ex2_approx(l0 - sb.x) * sc.x, ex2_approx(l1 - sb.y) * sc.y, ex2_approx(l2 - sb.z) * sc.z,
                                              ex2_approx(l3 - sb.w) * sc.w);
                float* row = dst + (size_t)q * pitch;
                if (e0 + 3 < n) {
                    *reinterpret_cast<float4*>(row) = gm;
                } else {
                    if (e0 < n) row[0] = gm.x;
                    if (e0 + 1 < n) row[1] = gm.y;
                    if (e0 + 2 < n) row[2] = gm.z;
                }
            }
        }
        mbar_arrive_after(&empty[sb2], dep);
    }
    if (mode == 0 || mode == 2) {
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 16);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 8);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 4);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 2);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 1);
        if (lane == 0) atomicAdd(ll_out, ll_acc);
    }
    }
}

// ===========================================================================
// Scoring of new events (gmm_score): the E-step's operand path and logits (tc_stage_operand / tc_split_rows /
// tc_tile_logits), with an epilogue that stores 12 B per event instead of 4 K: the label (argmax of the posterior,
// lowest k on ties, -1 when every logit is NaN), the top responsibility and the log-density (the E-step's denominator).
// Events are read from a chunk `x_aos` [n][D] of the caller's batch.
//   K <= 64: one launch (pass 0, last).  max_resp = ex2(l_max - M) * (1 / S), the E-step's operations for the stored
//            responsibility of that cluster, so it is bit-identical to it.
//   K > 64:  P launches for P passes of 64 clusters.  Passes 0 .. P-2 keep a per-event running (log-denominator, best
//            base-2 logit, best k) in run_*; the log-denominator is joined as the E-step's mode 2 joins it and an earlier
//            pass wins ties.  The last pass joins, stores the outputs and max_resp = exp(l_best - denominator).
// Every pass flags the chunk (*flag = 1) when an event has a coordinate that is not finite or lies beyond 2^14 global
// standard deviations (the bound tc_estep_range_ok applies to the training data: the FP16 event operand overflows).
// ===========================================================================
template <int D, int NSG>
__global__ void __launch_bounds__(ECfg<D>::THREADS, 1)
score_tc_kernel(const float* __restrict__ x_aos, const uint8_t* __restrict__ b_img, const float* __restrict__ ck,
                const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f, int n, int K, int kbase,
                int pass, int last, float* run_den, float* run_bl, int* run_bk, int* __restrict__ labels,
                float* __restrict__ max_resp, float* __restrict__ logp, double* __restrict__ ll_out, int* __restrict__ flag) {
    using C = ECfg<D>;
    constexpr int CP = C::CP;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
    const float* ck_s = reinterpret_cast<const float*>(smem + C::OFF_CK);
    const float* sh_s = reinterpret_cast<const float*>(smem + C::OFF_SH);
    const float* isc_s = sh_s + 32;

    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int gid = lane >> 2, qd = lane & 3;
    const int ntiles = (n + 63) / 64;
    tc_stage_operand<D>(smem, b_img, ck, shift_f, inv_scale_f, NSG);

    const int r0 = warp * 16 + gid;
    float2 xa[CP], xb[CP];
    auto load_rows = [&](int t) {
        const long long e0 = (long long)t * 64 + r0, e1 = e0 + 8;
#pragma unroll
        for (int j = 0; j < CP; j++) {
            xa[j] = e0 < n ? __ldg(reinterpret_cast<const float2*>(x_aos + (size_t)e0 * D + 8 * j + 2 * qd)) : make_float2(0.f, 0.f);
            xb[j] = e1 < n ? __ldg(reinterpret_cast<const float2*>(x_aos + (size_t)e1 * D + 8 * j + 2 * qd)) : make_float2(0.f, 0.f);
        }
    };
    const int stride = (int)gridDim.x * C::NWG;
    int t = (int)blockIdx.x * C::NWG + wg;
    if (t < ntiles) load_rows(t);
    const uint32_t ones = qd == 0 ? 0x3C003C00u : 0u;
    const uint32_t bsm = smem_u32(smem + C::OFF_B);
    double ll_acc = 0.0;
    constexpr float kLn2 = 0.6931471805599453f, kLog2e = 1.4426950408889634f;
    bool out_of_range = false;
    mbar_wait(b_full, 0);

    for (; t < ntiles; t += stride) {
        const long long e0 = (long long)t * 64 + r0, e1 = e0 + 8;
#pragma unroll
        for (int j = 0; j < CP; j++)
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const float2 x = r ? xb[j] : xa[j];
                const float z0 = __fmul_rn(__fsub_rn(x.x, sh_s[8 * j + 2 * qd]), isc_s[8 * j + 2 * qd]);
                const float z1 = __fmul_rn(__fsub_rn(x.y, sh_s[8 * j + 2 * qd + 1]), isc_s[8 * j + 2 * qd + 1]);
                out_of_range |= (r ? e1 : e0) < n && (!(fabsf(z0) <= 16384.0f) || !(fabsf(z1) <= 16384.0f));
            }
        uint32_t zh[CP][2], zl[CP][2];
        tc_split_rows<D>(xa, xb, sh_s, isc_s, qd, zh, zl);
        if (t + stride < ntiles) load_rows(t + stride);

        float lg[C::MAXSG][8];
        tc_tile_logits<D, NSG>(zh, zl, bsm, ck_s, qd, ones, lg);

        // per row: the E-step's max (fmaxf, from -FLT_MAX) and the arg-max over the pass's clusters, this lane's 16 logits
        // in increasing k, then the quad with (value, index) pairs; lowest k on ties, NaN logits never win
        float mx[2] = {-FLT_MAX, -FLT_MAX}, bl[2] = {-INFINITY, -INFINITY};
        int bk[2] = {-1, -1};
#pragma unroll
        for (int sg = 0; sg < C::MAXSG; sg++)
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const float l = lg[sg][u];
                const int k = sg * C::GB + 8 * (qd & 1) + 4 * (qd >> 1) + (u >> 1);
                mx[u & 1] = fmaxf(mx[u & 1], l);
                if (k < K && (l > bl[u & 1] || (bk[u & 1] < 0 && l == l))) { bl[u & 1] = l; bk[u & 1] = kbase + k; }
            }
#pragma unroll
        for (int r = 0; r < 2; r++) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bl[r], o);
                const int ok = __shfl_xor_sync(0xffffffffu, bk[r], o);
                if (ok >= 0 && (bk[r] < 0 || ov > bl[r] || (ov == bl[r] && ok < bk[r]))) { bl[r] = ov; bk[r] = ok; }
            }
        }
        // the denominator exactly as the E-step forms it
        float sm[2] = {0.f, 0.f};
#pragma unroll
        for (int sg = 0; sg < C::MAXSG; sg++)
#pragma unroll
            for (int u = 0; u < 8; u++) sm[u & 1] += ex2_approx(lg[sg][u] - mx[u & 1]);
        const long long er[2] = {e0, e1};
        float dx[2] = {0.f, 0.f}, pbl[2] = {0.f, 0.f};
        int pbk[2] = {-1, -1};
#pragma unroll
        for (int r = 0; r < 2; r++) {
            sm[r] += __shfl_xor_sync(0xffffffffu, sm[r], 1);
            sm[r] += __shfl_xor_sync(0xffffffffu, sm[r], 2);
            // the running state is updated in place: every lane reads before any writes
            if (pass > 0 && er[r] < n) { dx[r] = run_den[er[r]]; pbl[r] = run_bl[er[r]]; pbk[r] = run_bk[er[r]]; }
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 2; r++) {
            float denom = fmaf(mx[r], kLn2, logf(sm[r]));
            float mr = ex2_approx(bl[r] - mx[r]) * (1.0f / sm[r]);
            if (pass > 0) {
                const float g = fmaxf(fmaxf(denom, dx[r]), -FLT_MAX);
                const float tot = g + logf(__expf(denom - g) + __expf(dx[r] - g));
                // max_resp with the operations of the E-step's stored value: its mode 2 for a winner of this (last) pass,
                // its mode 3 for a winner of an earlier one (the product rounded on its own)
                if (bk[r] >= 0 && (pbk[r] < 0 || bl[r] > pbl[r])) {           // an earlier pass wins ties
                    const float sc = (1.0f / sm[r]) * __expf(denom - tot);
                    mr = ex2_approx(bl[r] - mx[r]) * sc;
                } else {
                    bl[r] = pbl[r]; bk[r] = pbk[r];
                    mr = ex2_approx(bl[r] - __fmul_rn(tot, kLog2e));
                }
                denom = tot;
            }
            if (qd == 0 && er[r] < n) {
                if (last) {
                    labels[er[r]] = bk[r];
                    max_resp[er[r]] = bk[r] >= 0 ? mr : __int_as_float(0x7fc00000);
                    logp[er[r]] = denom;
                    ll_acc += (double)denom;
                } else {
                    run_den[er[r]] = denom; run_bl[er[r]] = bl[r]; run_bk[er[r]] = bk[r];
                }
            }
        }
    }
    if (__any_sync(0xffffffffu, out_of_range) && lane == 0) *flag = 1;
    if (last) {
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 16);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 8);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 4);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 2);
        ll_acc = ll_acc + __shfl_down_sync(0xffffffffu, ll_acc, 1);
        if (lane == 0) atomicAdd(ll_out, ll_acc);
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
struct TcState {
    const float* d_x = nullptr;
    const float* d_x_soa = nullptr;
    DeviceArray<float> d_z_soa;      // [D][memb_pitch] centred/scaled SoA copy (M-step TMA source)
    float* d_memb = nullptr;
    size_t memb_pitch = 0;
    int n = 0, D = 0, Kmax = 0, num_sms = 132;
    CUtensorMap tm_x{}, tm_g{};
    bool maps_ok = false;
    DeviceArray<float> d_shift_f;    // [32]
    DeviceArray<float> d_inv_scale_f;   // [32]
    DeviceArray<double> d_scale;     // [32] = 1 / inv_scale_f (double)
    DeviceArray<float> d_scratch;    // [32-cluster blocks][ranges][MT][128][32] per-range partial sums, written once per launch
    bool have_shift = false;
    bool mstep_ready = false;        // the fixed-point quanta of the feature rows are set and inside the supported range
    float zmax[GMM_MAX_DIMENSIONS] = {0};    // power-of-two bound of |z_d| over the whole data set
    MMagic magic{0.f, 0.f};          // rounding constants of the coordinate / product rows
    DeviceArray<int3> d_rowmap;      // [MT * 128] operand row -> (packed statistic, dimension i, dimension j)
    DeviceArray<int> d_opmap;        // [MT * 128] operand row -> its factors a | b << 8 (mstep_row_layout)
    CUtensorMap tm_cx{}, tm_cg{};    // tc_launch_mstep_on: maps over the caller's chunk buffers, for cmap_n events
    const void* cmap_z = nullptr;
    const void* cmap_g = nullptr;
    size_t cmap_pitch = 0;
    int cmap_n = -1;
    // E-step
    CUtensorMap tm_x128{};
    bool emap_ok = false;
    uint8_t* d_bimg = nullptr;       // [MAXNG * B_GROUP] resident B operand image
    uint8_t* h_bimg = nullptr;       // pinned
    size_t bimg_bytes = 0;
    DeviceArray<uint8_t> d_opnd;     // [ck (e_ck_len floats) | B image]; d_ck / d_bimg point into it
    PinnedArray<uint8_t> h_opnd;     // mirror
    Event ev_h2d;                    // the last operand copy has left the pinned buffer
    bool h2d_pending = false;
    float* d_ck = nullptr;           // [passes][ck 64 | mult 64]: additive constant and quadratic-form multiplier per cluster
    float* h_ck = nullptr;           // pinned mirror
    DeviceArray<float> d_den;        // [memb_pitch] running / total log-denominator per event (Kmax > 64 only)
    int e_ck_len = 0;                // Kmax rounded up to whole passes of 64
    int e_NG = 0;
    int host_threads = 8;
    // cudaFuncAttributeMaxDynamicSharedMemorySize is per device: the "already set" flags live with the (per-device) state
    bool attr_estep = false, attr_mstep = false, attr_score = false;
    double h_shift[GMM_MAX_DIMENSIONS] = {0}, h_scale[GMM_MAX_DIMENSIONS] = {0};
};

static PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    return fn;
}

static int make_map_2d(CUtensorMap* m, const void* base, uint64_t dim0, uint64_t dim1, uint64_t stride1_bytes, uint32_t box0, uint32_t box1,
                       bool swizzle128 = false) {
    auto fn = encode_fn();
    if (!fn) return fail(GMM_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[2] = {dim0, dim1};
    cuuint64_t strides[1] = {stride1_bytes};
    cuuint32_t box[2] = {box0, box1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(GMM_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return GMM_OK;
}

bool tc_mstep_supported(int D, int K) {
    (void)K;
    return D == 4 || D == 8 || D == 12 || D == 16 || D == 20 || D == 24;
}
bool tc_estep_supported(int D, int K) { return (D == 8 || D == 16 || D == 24) && K >= 1 && K <= GMM_MAX_CLUSTERS; }

// bytes of the B image of one pass (64 clusters = MAXSG supergroups)
template <int D> static size_t ecfg_pass_bytes() { return (size_t)ECfg<D>::MAXSG * ECfg<D>::B_SG; }
static size_t pass_bytes_for(int D) {
    switch (D) { case 8: return ecfg_pass_bytes<8>(); case 16: return ecfg_pass_bytes<16>(); case 24: return ecfg_pass_bytes<24>(); default: return 0; }
}

int tc_create(TcState** out, const float* d_x_aos, const float* d_x_soa, int n, int D, int Kmax, float* d_memb, size_t memb_pitch, int num_sms,
              cudaStream_t stream) {
    (void)stream;
    TcState* t = new TcState();
    t->d_x = d_x_aos; t->d_x_soa = d_x_soa; t->d_memb = d_memb; t->memb_pitch = memb_pitch; t->n = n; t->D = D; t->Kmax = Kmax; t->num_sms = num_sms;
    *out = t;
    if (n <= 0 || !tc_mstep_supported(D, Kmax)) return GMM_OK;
    if (int rc = t->d_shift_f.reserve(GMM_MAX_DIMENSIONS)) return rc;
    if (int rc = t->d_inv_scale_f.reserve(GMM_MAX_DIMENSIONS)) return rc;
    if (int rc = t->d_scale.reserve(GMM_MAX_DIMENSIONS)) return rc;
    // tensor maps: SoA events [D][pitch] viewed as (events, dims) -> smem tile [D][32 events] (SWIZZLE_128B);
    // responsibilities [Kmax][pitch] viewed as (events, clusters)
    if (int rc = t->d_z_soa.reserve(memb_pitch * D)) return rc;
    if (int rc = make_map_2d(&t->tm_x, t->d_z_soa, (uint64_t)n, (uint64_t)D, (uint64_t)memb_pitch * 4, kTE, (uint32_t)D, /*swizzle128=*/true)) return rc;
    if (int rc = make_map_2d(&t->tm_g, d_memb, (uint64_t)n, (uint64_t)Kmax, (uint64_t)memb_pitch * 4, kTE, kNCL, /*swizzle128=*/true)) return rc;
    t->maps_ok = true;
    if (D == 8 || D == 16 || D == 24) {
        const int passes = (Kmax + 63) / 64;
        t->e_ck_len = passes * 64;
        t->bimg_bytes = (size_t)passes * pass_bytes_for(D);
        // one staging / device buffer [ck | B image]: the operand of an iteration travels in ONE H2D copy
        const size_t ck_bytes = sizeof(float) * 2 * t->e_ck_len;     // 512 B per pass: keeps the image 16-byte aligned
        if (int rc = t->d_opnd.reserve(ck_bytes + t->bimg_bytes)) return rc;
        if (int rc = t->h_opnd.reserve(ck_bytes + t->bimg_bytes)) return rc;
        t->d_ck = reinterpret_cast<float*>(t->d_opnd.get());
        t->h_ck = reinterpret_cast<float*>(t->h_opnd.get());
        t->d_bimg = t->d_opnd + ck_bytes;
        t->h_bimg = t->h_opnd + ck_bytes;
        if (int rc = t->ev_h2d.create(cudaEventDisableTiming)) return rc;
        if (passes > 1)
            if (int rc = t->d_den.reserve(memb_pitch)) return rc;
        t->emap_ok = true;
    }
    const int mt = mstep_tiles(D);
    {
        // operand row -> (packed statistic, dimension i, dimension j) for the finalisation, and its two factors for the kernel
        const std::vector<MRow> rows = mstep_row_layout(D);
        if (rows.size() != (size_t)mt * 128) return fail(GMM_ERR_STATE, "tensor M-step row map: the statistics do not fit the feature tiles");
        std::vector<int3> rm(rows.size());
        std::vector<int> om(rows.size());
        std::vector<char> seen((size_t)num_features(D), 0);
        for (size_t row = 0; row < rows.size(); row++) {
            const MRow& r = rows[row];
            rm[row] = make_int3(r.f, r.i, r.j);
            om[row] = r.a | r.b << 8;
            if (r.f >= 0) {
                if (seen[r.f]) return fail(GMM_ERR_STATE, "tensor M-step row map: a statistic is produced twice");
                seen[r.f] = 1;
            }
        }
        for (char c : seen) if (!c) return fail(GMM_ERR_STATE, "tensor M-step row map: a statistic is not produced");
        if (int rc = t->d_rowmap.reserve(rm.size())) return rc;
        CUDA_TRY(cudaMemcpy(t->d_rowmap, rm.data(), sizeof(int3) * rm.size(), cudaMemcpyHostToDevice));
        if (int rc = t->d_opmap.reserve(om.size())) return rc;
        CUDA_TRY(cudaMemcpy(t->d_opmap, om.data(), sizeof(int) * om.size(), cudaMemcpyHostToDevice));
    }
    const int ytiles = (Kmax + 63) / 64 * (64 / kNCL);         // 32-cluster column blocks of whole 64-cluster CTAs
    return t->d_scratch.reserve((size_t)num_sms * ytiles * mt * 128 * kNCL);
}

void tc_set_host_threads(TcState* t, int n) { if (t) t->host_threads = n < 1 ? 1 : n; }
bool tc_mstep_ready(const TcState* t) { return t && t->maps_ok && t->have_shift && t->mstep_ready; }
bool tc_estep_range_ok(const TcState* t) {
    if (!t || !t->have_shift) return false;
    for (int d = 0; d < t->D; d++)
        if (!(t->zmax[d] <= 16384.0f)) return false;
    return true;
}

void tc_destroy(TcState* t) { delete t; }

int tc_set_shift_scale(TcState* t, double* shift, const double* scale, const double* xmin, const double* xmax, cudaStream_t stream) {
    if (!t || !t->maps_ok) return GMM_OK;
    float sf[GMM_MAX_DIMENSIONS] = {0}, isf[GMM_MAX_DIMENSIONS] = {0};
    double sc[GMM_MAX_DIMENSIONS] = {0};
    for (int d = 0; d < t->D; d++) {
        sf[d] = (float)shift[d];
        shift[d] = (double)sf[d];                       // the host finalisation must use the value the kernel used
        const double s = (scale && scale[d] > 0) ? scale[d] : 1.0;
        isf[d] = (float)(1.0 / s);
        sc[d] = 1.0 / (double)isf[d];
        t->h_shift[d] = shift[d];
        t->h_scale[d] = sc[d];
        // power-of-two bound of |z_d| = |(x - shift) * inv_scale| over the data (float arithmetic of the kernels + slack)
        const double za = std::fmax(std::fabs(xmax[d] - (double)sf[d]), std::fabs(xmin[d] - (double)sf[d])) * (double)isf[d] * (1.0 + 1e-6);
        int e2 = 0;
        if (za > 0 && std::isfinite(za)) { e2 = std::ilogb(za) + 1; }      // za < 2^e2
        t->zmax[d] = std::isfinite(za) ? (float)std::ldexp(1.0, e2) : INFINITY;
    }
    // Fixed-point quanta of the M-step feature rows: q = bound * 2^-11, magic = 1.5 * 2^23 * q, bound = the power-of-two
    // bound of |z| over all dimensions (squared for the product rows).  Data with outliers beyond 64 standard deviations
    // would leave too few bits below the quantum for the bulk of the events: such a data set is served by the FP64
    // SIMT M-step instead (tc_mstep_ready() false; GMM_PATH_TENSOR reports it).
    {
        float zb = 0.f;
        for (int d = 0; d < t->D; d++) zb = std::fmax(zb, t->zmax[d]);
        t->mstep_ready = zb <= 64.0f;                              // false for inf / nan too
        const double q = (double)zb / (double)(1 << kPhiBits);
        t->magic.lin = (float)(1.5 * 8388608.0 * q);
        t->magic.prod = (float)(1.5 * 8388608.0 * q * (double)zb);
    }
    CUDA_TRY(cudaMemcpyAsync(t->d_shift_f, sf, sizeof(sf), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(t->d_inv_scale_f, isf, sizeof(isf), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(t->d_scale, sc, sizeof(sc), cudaMemcpyHostToDevice, stream));
    {
        dim3 grid((unsigned)std::min<long long>(4LL * t->num_sms, ((long long)t->n + 255) / 256), (unsigned)t->D);
        standardise_soa_kernel<<<grid, 256, 0, stream>>>(t->d_x_soa, t->d_z_soa, t->memb_pitch, t->n, t->D, t->d_shift_f, t->d_inv_scale_f);
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(stream));         // the staging arrays live on this stack frame
    t->have_shift = true;
    return GMM_OK;
}

// Host side of the tensor E-step operand: per cluster the upper-triangular factor W of
// Rinv = W^T W (Cholesky of the symmetrised inverse covariance, double), expressed in the
// centred/scaled coordinates of the kernel, FP16 hi/lo split, laid out as the resident
// K-major B image ([supergroup][block][chunk][128 rows][16 B]).  Fails (GMM_ERR_STATE) when Rinv
// is not positive definite or the factor overflows FP16; the caller then uses the SIMT kernel
// for this state.

// float -> IEEE half bits, round to nearest even (normal, subnormal and zero; callers check the range)
static inline uint16_t f2h_bits(float f) {
    uint32_t x;
    std::memcpy(&x, &f, 4);
    const uint32_t sign = (x >> 16) & 0x8000u;
    x &= 0x7fffffffu;
    if (x >= 0x47800000u) return (uint16_t)(sign | 0x7c00u);
    if (x < 0x38800000u) {                      // below the smallest normal half: value * 2^24, rounded
        float a;
        std::memcpy(&a, &x, 4);
        return (uint16_t)(sign | (uint32_t)lrintf(a * 16777216.0f));
    }
    x += ((x >> 13) & 1u) + 0xfffu;
    return (uint16_t)(sign | ((x - 0x38000000u) >> 13));
}
static inline float h2f_bits(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    const uint32_t em = h & 0x7fffu;
    float r;
    if (em >= 0x0400u) {                         // normal (inf/nan never produced here)
        const uint32_t x = sign | ((em << 13) + 0x38000000u);
        std::memcpy(&r, &x, 4);
    } else {
        r = (float)em * (1.0f / 16777216.0f);
        if (sign) r = -r;
    }
    return r;
}

// Operand rows of cluster k (k >= K: padding cluster of the last supergroup).  Returns 0, 1 (Rinv not positive
// definite) or 2 (factor outside the FP16 range).  Clusters are independent: callers may run this in parallel.
// Wext (optional): the upper-triangular factor W with Rinv = W^T W already computed by the caller in double (row-major
// [D][D]); otherwise it is derived here from host->Rinv.
template <int D>
static int bimg_cluster(TcState* t, const clusters_t* host, int k, int K, const double* Wext = nullptr) {
    using C = ECfg<D>;
    int bad = 0;
    {
        const int sg = k / C::GB, i = k % C::GB;
        // 16-byte K-chunk `chunk` of output column d of this cluster: K-major SWIZZLE_NONE image
        // [supergroup][block c = d/8][chunk][N = 16 clusters x 8 columns][16 B]
        auto rowp = [&](int d, int chunk) -> uint16_t* {
            const int c = d / 8, ncol = i * 8 + (d % 8);
            return reinterpret_cast<uint16_t*>(t->h_bimg + ((size_t)sg * C::CP + c) * C::B_BLOCK + (size_t)chunk * C::N * 16 + (size_t)ncol * 16);
        };
        if (k >= K) {                                    // padding cluster of the last supergroup: all-zero rows
            for (int d = 0; d < D; d++)
                for (int c = 0; c < C::NCHKB; c++) std::memset(rowp(d, c), 0, 16);
            return 0;
        }
        double A[D][D], Gc[D][D];
        const float* Ri = host->Rinv + (size_t)k * D * D;
        bool ok = true;
        if (Wext) {                                      // W = Gc^T
            for (int r = 0; r < D; r++)
                for (int j = 0; j < D; j++) Gc[r][j] = Wext[j * D + r];
        } else {
            for (int r = 0; r < D; r++)
                for (int j = 0; j < D; j++) { A[r][j] = 0.5 * ((double)Ri[r * D + j] + (double)Ri[j * D + r]); Gc[r][j] = 0.0; }
        }
        for (int j = 0; j < D && !Wext; j++) {                    // right-looking Cholesky A = Gc Gc^T (axpy updates vectorise)
            const double d = A[j][j];
            if (!(d > 0.0) || !std::isfinite(d)) { ok = false; break; }
            const double piv = std::sqrt(d), rp = 1.0 / piv;
            Gc[j][j] = piv;
            for (int r = j + 1; r < D; r++) Gc[r][j] = A[r][j] * rp;
            for (int r = j + 1; r < D; r++) {
                const double l = Gc[r][j];
                for (int cc = j + 1; cc <= r; cc++) A[r][cc] -= l * Gc[cc][j];
            }
        }
        if (!ok) return 1;
        // rows of W = Gc^T in the kernel's coordinates:  y_d = sum_j W'[d][j] z_j + v_d,  W'[d][j] = Gc[j][d] * scale_j (j >= d)
        alignas(32) float wrow[D][D];
        double vd[D];
        float amax = 0.f;
        for (int d = 0; d < D; d++) {
            double v = 0.0;
            for (int j = 0; j < D; j++) {
                const double w = (j >= d) ? Gc[j][d] : 0.0;
                v = std::fma(-w, (double)host->means[(size_t)k * D + j] - t->h_shift[j], v);   // finalize_params_kernel: the same fused steps
                wrow[d][j] = (float)(w * t->h_scale[j]);
                amax = std::fmax(amax, std::fabs(wrow[d][j]));
            }
            vd[d] = v;
            amax = std::fmax(amax, (float)std::fabs(v));
        }
        if (!std::isfinite(amax)) return 2;
        // Per-cluster power-of-two scale: the largest operand entry lands in [2^12, 2^13) whatever the width of the
        // cluster (a cluster of relative width 1e-4 has factors ~1e4 - 1e5 and used to leave the FP16 range; a very wide
        // one pushed its lo parts into the FP16 subnormals).  The epilogue divides the squared norm by scale^2 (exact).
        int e2 = amax > 0.f ? 12 - std::ilogb(amax) : 0;
        e2 = e2 > 40 ? 40 : (e2 < -40 ? -40 : e2);
        for (int d = 0; d < D; d++) {
            for (int j = 0; j < D; j++) wrow[d][j] = std::ldexp(wrow[d][j], e2);
            vd[d] = std::ldexp(vd[d], e2);
            for (int c = 0; c < C::CP; c++) {
                uint16_t *ph = rowp(d, c), *pl = rowp(d, C::CP + c);      // x (zh_c, zl_c) [aliased], x zh_c
#if defined(__F16C__) && defined(__AVX__)
                const __m256 w8 = _mm256_load_ps(&wrow[d][8 * c]);
                const __m128i h8 = _mm256_cvtps_ph(w8, _MM_FROUND_TO_NEAREST_INT | _MM_FROUND_NO_EXC);
                const __m256 l8 = _mm256_sub_ps(w8, _mm256_cvtph_ps(h8));  // exact: hi is w rounded to 11 bits
                _mm_storeu_si128(reinterpret_cast<__m128i*>(ph), h8);
                _mm_storeu_si128(reinterpret_cast<__m128i*>(pl), _mm256_cvtps_ph(l8, _MM_FROUND_TO_NEAREST_INT | _MM_FROUND_NO_EXC));
#else
                for (int e = 0; e < 8; e++) {
                    const uint16_t wh = f2h_bits(wrow[d][8 * c + e]);
                    ph[e] = wh;
                    pl[e] = f2h_bits(wrow[d][8 * c + e] - h2f_bits(wh));
                }
#endif
            }
            const float vf = (float)vd[d];
            if (!(std::fabs(vf) < 6.0e4f)) bad = 2;
            uint16_t* pv = rowp(d, 2 * C::CP);
            const uint16_t vh = f2h_bits(vf);
            std::memset(pv, 0, 16);
            pv[0] = vh;
            pv[1] = f2h_bits((float)(vd[d] - (double)h2f_bits(vh)));
            if (C::NCHKB > 2 * C::CP + 1) std::memset(rowp(d, 2 * C::CP + 1), 0, 16);
        }
        float* ckp = t->h_ck + (size_t)(k / 64) * 128 + (k % 64);
        ckp[0] = host->constant[k] + (float)std::log((double)host->pi[k]);   // additive term of estep1 (gaussian_kernel.cu:442); ln pi in double, as on the device
        ckp[64] = (float)std::ldexp(-0.5 * 1.4426950408889634, -2 * e2);
    }
    return bad;
}

static int bimg_cluster_any(TcState* t, const clusters_t* host, int k, int K, const double* Wext = nullptr) {
    switch (t->D) {
        case 8: return bimg_cluster<8>(t, host, k, K, Wext);
        case 16: return bimg_cluster<16>(t, host, k, K, Wext);
        case 24: return bimg_cluster<24>(t, host, k, K, Wext);
        default: return 3;
    }
}

int tc_params_begin(TcState* t, int K, cudaStream_t stream) {
    if (!t || !t->emap_ok) return fail(GMM_ERR_STATE, "tensor E-step not initialised for this shape");
    if (!t->have_shift) return fail(GMM_ERR_STATE, "tensor E-step needs the global moments (shift/scale) first");
    (void)stream;
    if (t->h2d_pending) {                                // the previous copy out of the pinned buffer must have finished
        CUDA_TRY(cudaEventSynchronize(t->ev_h2d));
        t->h2d_pending = false;
    }
    for (int k = K; k < t->e_ck_len; k++) {               // padding clusters: never win the log-sum-exp
        float* ckp = t->h_ck + (size_t)(k / 64) * 128 + (k % 64);
        ckp[0] = -1e30f;
        ckp[64] = 0.f;
    }
    return GMM_OK;
}
int tc_params_padded(const TcState*, int K) { return (K + 15) / 16 * 16; }
int tc_params_cluster(TcState* t, const clusters_t* host, int k, int K) { return bimg_cluster_any(t, host, k, K); }
int tc_params_cluster_w(TcState* t, const clusters_t* host, int k, int K, const double* W) { return bimg_cluster_any(t, host, k, K, W); }
int tc_params_commit(TcState* t, int K, int bad, cudaStream_t stream) {
    if (bad == 1) return fail(GMM_ERR_STATE, "tensor E-step: inverse covariance of a cluster is not positive definite");
    if (bad == 2) return fail(GMM_ERR_STATE, "tensor E-step: whitening factor exceeds the FP16 range");
    if (bad) return fail(GMM_ERR_ARG, "tensor E-step: unsupported D");
    t->e_NG = (K + 15) / 16;
    // only the supergroups in use travel (the image is contiguous per supergroup; 4 supergroups = 64 clusters)
    const size_t used = (size_t)t->e_NG * (pass_bytes_for(t->D) / 4);
    CUDA_TRY(cudaMemcpyAsync(t->d_opnd, t->h_opnd, sizeof(float) * 2 * t->e_ck_len + used, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaEventRecord(t->ev_h2d, stream));
    t->h2d_pending = true;
    return GMM_OK;
}


int tc_upload_params(TcState* t, const clusters_t* host, int K, cudaStream_t stream) {
    if (int rc = tc_params_begin(t, K, stream)) return rc;
    const int kp = tc_params_padded(t, K);
    const int nt = t->host_threads;
    int bad = 0;
    (void)nt;
#pragma omp parallel for schedule(static) num_threads(nt) reduction(max : bad) if (nt > 1 && K >= 8)
    for (int k = 0; k < kp; k++) {
        const int b = tc_params_cluster(t, host, k, K);
        bad = b > bad ? b : bad;
    }
    return tc_params_commit(t, K, bad, stream);
}

// ===========================================================================
// Device-side M-step finalisation (one CTA per cluster): everything the host does between the reduced statistics
// and the next E-step — N, means, R (gaussian.cu:611-622, 663-679 with the rules of mstep_covariance1,
// gaussian_kernel.cu:658-675), inverse + constant + pi (constants_kernel, :172-259) and the E-step's resident
// operand (bimg_cluster above) — so that an EM iteration needs no device -> host -> device round trip
// (D2H of the statistics, thread-team wake-up, H2D of the operand).  The same operations in the same order as
// host_math.cpp (double, results stored as float): reverse Cholesky R = U U^T, W = U^-1, Rinv = W^T W,
// ln det R = 2 sum ln U_ii, so that the device and the host finalisation produce bit-identical parameter sets and
// E-step operands (EM amplifies any last-bit difference between the two).  A cluster the host would NOT serve this way (R not positive definite, factor outside FP16)
// is not handled here: the kernel records the iteration in bad[0] (first failure wins), every later launch returns
// immediately, and the host replays from the last good parameter set through its own path (gmm_api.cu).
// Parameter set layout (floats, stride Kmax): N | pi | constant | means [Kmax][D] | R [Kmax][D][D] | Rinv [Kmax][D][D].
// ===========================================================================
__host__ __device__ inline size_t pset_off_means(int Kmax) { return 3 * (size_t)Kmax; }
__host__ __device__ inline size_t pset_off_R(int Kmax, int D) { return pset_off_means(Kmax) + (size_t)Kmax * D; }
__host__ __device__ inline size_t pset_off_Rinv(int Kmax, int D) { return pset_off_R(Kmax, D) + (size_t)Kmax * D * D; }

#ifdef GMM_FIN_PROF   // build-time phase stamps of finalize_params_kernel (CTA 0, thread 0 prints cycle deltas); off by default
#define FIN_STAMP(i) do { if (k == 0 && tid == 0) fin_t[i] = clock64(); } while (0)
#else
#define FIN_STAMP(i) do { } while (0)
#endif

template <int D> struct FinCfg { static constexpr int T = (D * D > 256 ? (D * D + 31) / 32 * 32 : 256), NW = T / 32; };   // a thread per matrix element

template <int D>
__global__ void __launch_bounds__(FinCfg<D>::T)
finalize_params_kernel(const double* __restrict__ stats, const float* __restrict__ avgvar, const float* __restrict__ shift_f,
                       const double* __restrict__ scale, float* __restrict__ set, int Kmax, int K, int kp,
                       uint8_t* __restrict__ bimg, float* __restrict__ ck, double* __restrict__ ll_out, int* __restrict__ bad, int iter,
                       int fault_iter) {
    // Latency-bound by construction (one CTA works through a 24 x 24 factorisation, 64 CTAs on 132 SMs): one global round trip
    // (the cluster's statistics row is staged in shared memory), then the host's factorisation and inverse with a thread per row /
    // column (see below), and a thread per matrix element for everything else.
#ifdef GMM_FIN_PROF
    long long fin_t[10];
#endif
    using C = ECfg<D>;
    constexpr int T = FinCfg<D>::T, NW = FinCfg<D>::NW;
    constexpr int F = 1 + D + D * (D + 1) / 2;
    constexpr int LD = D + 1;
    const int k = blockIdx.x, tid = threadIdx.x;
    if (bad[0] >= 0) return;                                   // an earlier iteration failed: leave the last good state alone
    float* ckp = ck + (size_t)(k / 64) * 128 + (k % 64);
    const int sg = k / C::GB, ci = k % C::GB;
    auto rowp = [&](int d, int chunk) -> uint8_t* {            // 16-byte K chunk `chunk` of output column d (see bimg_cluster)
        return bimg + ((size_t)sg * C::CP + d / 8) * C::B_BLOCK + (size_t)chunk * C::N * 16 + (size_t)(ci * 8 + d % 8) * 16;
    };
    if (k >= K) {                                              // padding: never wins the log-sum-exp, all-zero operand rows
        if (tid == 0) { ckp[0] = -1e30f; ckp[64] = 0.f; }
        if (k < kp)
            for (int idx = tid; idx < D * C::NCHKB; idx += T) *reinterpret_cast<uint4*>(rowp(idx / C::NCHKB, idx % C::NCHKB)) = make_uint4(0u, 0u, 0u, 0u);
        return;
    }
    FIN_STAMP(0);
    __shared__ double sS[F + 3], sA[D][LD], sU[D][LD], sW[D][LD], sdm[D], sscale[D], svd[D], sredd[NW], ssumN;
    __shared__ float swr[D][LD], sredf[NW], sN[GMM_MAX_CLUSTERS];
    __shared__ int sbad;
    // ---- stage: the statistics row, the N = (float)S0 of every cluster (pi), shift / scale ----
    const double* s = stats + (size_t)k * F;
    for (int f = tid; f < F; f += T) sS[f] = s[f];
    for (int kk = tid; kk < K; kk += T) sN[kk] = (float)stats[(size_t)kk * F];
    double shift_d = 0.0;
    if (tid < D) { shift_d = (double)shift_f[tid]; sscale[tid] = scale[tid]; }
    const float av = avgvar[k];
    double ll_slot = 0.0;
    if (k == 0 && tid == 0) ll_slot = stats[(size_t)K * F];
    if (tid == 0) sbad = 0;
    __syncthreads();
    FIN_STAMP(1);
    const double S0 = sS[0];
    const float Nf = (float)S0;
    if (k == 0 && tid == 0) {
        *ll_out = ll_slot;                                     // log-likelihood of the E-step these statistics came from
        if (isnan(S0)) atomicMax(&sbad, 4);                    // the all-reduce kernel marks a failed exchange with NaN
        if (iter == fault_iter) atomicMax(&sbad, 1);           // test hook (option "finalize_fault_iter"): exercise the host replay
    }
    // ---- means (gaussian.cu:611-622), R (:663-679, gaussian_kernel.cu:658-675); pi after the inverse (see below) ----
    if (tid < D) {
        const double m = (S0 != 0.0) ? sS[1 + tid] / S0 : 0.0;
        const float mu = (Nf > 0.5f) ? (float)(m + shift_d) : 0.0f;
        sdm[tid] = (double)mu - shift_d;                       // mu - shift as the operand rows need it
        set[pset_off_means(Kmax) + (size_t)k * D + tid] = mu;
    }
    {
        float* R = set + pset_off_R(Kmax, D) + (size_t)k * D * D;
        const double inv = 1.0 / (double)Nf;
        for (int idx = tid; idx < D * D; idx += T) {
            const int i = idx / D, j = idx % D;
            if (j > i) continue;
            float v;
            if (Nf > 0.5f) {
                const double mi = (S0 != 0.0) ? sS[1 + i] / S0 : 0.0;
                double cov = (Nf >= 1.0f) ? fma(-mi, sS[1 + j], sS[1 + D + i * (i + 1) / 2 + j]) : 0.0;   // finalize_cluster: the same fused step
                if (i == j) cov += av;
                v = (float)(cov * inv);
            } else {
                v = (i == j) ? 1.0f : 0.0f;
            }
            R[i * D + j] = v; R[j * D + i] = v;
            sA[j][i] = (double)v;                              // upper triangle (row <= column) is what the factorisation reads
            if (i == j) sW[i][i] = 0.0; else { sW[j][i] = 0.0; sW[i][j] = 0.0; }
        }
    }
    __syncthreads();
    FIN_STAMP(2);
    // ---- R = U U^T from the last column (reverse Cholesky), then W = U^-1: the operations and their order of
    //      constants_cluster_spd (host_math.cpp), every product rounded before it is subtracted (__dmul_rn / __dsub_rn,
    //      as the host is compiled), correctly rounded sqrt and division — the device and the host finalisation give
    //      bit-identical factors.  Column j: thread i <= j forms its dot product over the finished columns m > j
    //      (thread j's is the pivot, which every thread recomputes), ONE barrier per column ----
    bool ok = true;
    for (int j = D - 1; j >= 0; j--) {
        double d = sA[j][j];
        for (int m = j + 1; m < D; m++) d = __dsub_rn(d, __dmul_rn(sU[j][m], sU[j][m]));
        if (!(d > 0.0) || !isfinite(d)) { ok = false; break; }    // the same value in every thread
        const double piv = sqrt(d), rp = 1.0 / piv;
        if (tid < j) {
            double v = sA[tid][j];
            for (int m = j + 1; m < D; m++) v = __dsub_rn(v, __dmul_rn(sU[tid][m], sU[j][m]));
            sU[tid][j] = __dmul_rn(v, rp);
        } else if (tid == j) {
            sU[j][j] = piv;
        }
        __syncthreads();
    }
    if (!ok) {
        if (tid == 0) { atomicCAS(&bad[0], -1, iter); atomicMax(&bad[1], 1); }
        return;
    }
    FIN_STAMP(3);
    // ---- W = U^-1 (upper triangular), a thread per column j: W[i][j] = -(sum_{m=i+1..j} U[i][m] W[m][j]) / U[i][i] ----
    if (tid < D) {
        const int j = tid;
        for (int i = D - 1; i > j; i--) sW[i][j] = 0.0;
        sW[j][j] = 1.0 / sU[j][j];
        for (int i = j - 1; i >= 0; i--) {
            double v = 0.0;
            for (int m = i + 1; m <= j; m++) v = __dsub_rn(v, __dmul_rn(sU[i][m], sW[m][j]));
            sW[i][j] = v / sU[i][i];
        }
    }
    if (tid == T - 1) {                                        // (a warp of its own, idle in this phase)
        // sum N[k] in the host's order (mixing_weights: k = 0, 1, ...): a double sum of floats that differ by many orders of
        // magnitude depends on its order, and pi must be the host's bit for bit (compute_pi, gaussian_kernel.cu:172-193)
        double sum = 0.0;
        for (int kk = 0; kk < K; kk++) sum += (double)sN[kk];
        ssumN = sum;
    }
    __syncthreads();
    FIN_STAMP(4);
    const float pik = Nf < 0.5f ? 1e-10f : (float)((double)Nf / ssumN);
    // ---- Rinv = W^T W, ln det, constant (gaussian_kernel.cu:241), N, pi; operand rows: W'[d][j] = W[d][j] * scale_j, v = -W (mu - shift) ----
    {
        float* Ri = set + pset_off_Rinv(Kmax, D) + (size_t)k * D * D;
        for (int idx = tid; idx < D * D; idx += T) {
            const int i = idx / D, j = idx % D;
            if (j < i) continue;
            double v = 0.0;
#pragma unroll 4
            for (int m = 0; m <= i; m++) v = __dadd_rn(v, __dmul_rn(sW[m][i], sW[m][j]));
            Ri[i * D + j] = (float)v; Ri[j * D + i] = (float)v;
        }
    }
    FIN_STAMP(5);
    float amax = 0.f;
    for (int idx = tid; idx < D * D; idx += T) {
        const int d = idx / D, j = idx % D;
        const float w = (j >= d) ? (float)(sW[d][j] * sscale[j]) : 0.f;
        swr[d][j] = w;
        amax = fmaxf(amax, fabsf(w));
    }
    if (tid >= 64 && tid < 64 + D) {                              // (a warp of its own: the row sums are serial)
        const int d = tid - 64;
        double v = 0.0;
#pragma unroll 4
        for (int j = d; j < D; j++) v = fma(-sW[d][j], sdm[j], v);     // bimg_cluster: the same fused steps
        svd[d] = v;
        amax = fmaxf(amax, (float)fabs(v));
    }
    if (tid == 32) {                                           // sum ln U_jj in the host's order
        double ld = 0.0;
        for (int j = D - 1; j >= 0; j--) ld += log(sU[j][j]);
        sredd[0] = ld;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((tid & 31) == 0) sredf[tid >> 5] = amax;
    __syncthreads();
    FIN_STAMP(6);
    const double ld = sredd[0];                                // sum ln U_jj
    const float cst = (float)(-D * 0.5 * log(2.0 * 3.1415926535897931) - 0.5 * (2.0 * ld));
    if (tid == 0) { set[k] = Nf; set[Kmax + k] = pik; set[2 * (size_t)Kmax + k] = cst; }
    amax = 0.f;
#pragma unroll
    for (int w = 0; w < NW; w++) amax = fmaxf(amax, sredf[w]);
    if (!isfinite(amax)) {
        if (tid == 0) { atomicCAS(&bad[0], -1, iter); atomicMax(&bad[1], 2); }
        return;
    }
    // per-cluster power-of-two scale: the largest operand entry lands in [2^12, 2^13) (see bimg_cluster)
    int e2 = amax > 0.f ? 12 - ilogbf(amax) : 0;
    e2 = e2 > 40 ? 40 : (e2 < -40 ? -40 : e2);
    for (int idx = tid; idx < D * C::CP; idx += T) {
        const int d = idx / C::CP, c = idx % C::CP;
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const float w0 = ldexpf(swr[d][8 * c + 2 * e], e2), w1 = ldexpf(swr[d][8 * c + 2 * e + 1], e2);
            const __half2 h = __floats2half2_rn(w0, w1);
            const float2 hf = __half22float2(h);
            hi[e] = *reinterpret_cast<const uint32_t*>(&h);
            lo[e] = pack_half2(w0 - hf.x, w1 - hf.y);          // exact difference: hi is w rounded to 11 bits
        }
        *reinterpret_cast<uint4*>(rowp(d, c)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);             // x (zh_c, zl_c) [aliased]
        *reinterpret_cast<uint4*>(rowp(d, C::CP + c)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);     // x zh_c
    }
    if (tid >= 128 && tid < 128 + D) {
        const int d = tid - 128;
        const double vs = ldexp(svd[d], e2);
        const float vf = (float)vs;
        if (!(fabsf(vf) < 6.0e4f)) atomicMax(&sbad, 2);
        const __half vh = __float2half_rn(vf);
        const __half vl = __float2half_rn((float)(vs - (double)__half2float(vh)));
        const uint32_t p = (uint32_t)__half_as_ushort(vh) | ((uint32_t)__half_as_ushort(vl) << 16);
        *reinterpret_cast<uint4*>(rowp(d, 2 * C::CP)) = make_uint4(p, 0u, 0u, 0u);
        if (C::NCHKB > 2 * C::CP + 1) *reinterpret_cast<uint4*>(rowp(d, 2 * C::CP + 1)) = make_uint4(0u, 0u, 0u, 0u);
    }
    if (tid == 0) {
        ckp[0] = cst + (float)log((double)pik);                // additive term of estep1 (gaussian_kernel.cu:442); ln pi as on the host
        ckp[64] = (float)ldexp(-0.5 * 1.4426950408889634, -2 * e2);
    }
    __syncthreads();
    FIN_STAMP(7);
#ifdef GMM_FIN_PROF
    if (k == 0 && tid == 0)
        printf("fin phases (cycles): stage %lld  means+R %lld  cholesky %lld  inverse %lld  Rinv %lld  rows+v+log %lld  operand %lld\n",
               fin_t[1] - fin_t[0], fin_t[2] - fin_t[1], fin_t[3] - fin_t[2], fin_t[4] - fin_t[3], fin_t[5] - fin_t[4], fin_t[6] - fin_t[5], fin_t[7] - fin_t[6]);
#endif
    if (tid == 0 && sbad) { atomicCAS(&bad[0], -1, iter); atomicMax(&bad[1], sbad); }
}

size_t tc_param_set_floats(int Kmax, int D) { return (size_t)Kmax * (3 + (size_t)D + 2 * (size_t)D * D); }
size_t tc_param_set_off(int Kmax, int D, int which) {
    switch (which) {
        case 0: return 0;                                   // N
        case 1: return (size_t)Kmax;                        // pi
        case 2: return 2 * (size_t)Kmax;                    // constant
        case 3: return pset_off_means(Kmax);
        case 4: return pset_off_R(Kmax, D);
        default: return pset_off_Rinv(Kmax, D);
    }
}
bool tc_finalize_supported(const TcState* t, int K) {
    return t && t->emap_ok && t->have_shift && tc_estep_supported(t->D, K) && tc_estep_range_ok(t);
}
int tc_launch_finalize(TcState* t, int K, const double* d_stats, const float* d_avgvar, float* d_set, double* d_ll, int* d_bad, int iter,
                       int fault_iter, cudaStream_t stream) {
    if (!tc_finalize_supported(t, K)) return fail(GMM_ERR_STATE, "device-side finalisation not available for this state");
    const int kp = tc_params_padded(t, K);
    const int grid = ((K + 63) / 64) * 64;                     // whole passes: the padding clusters of the last pass get their constants
#define GMM_FIN(d) finalize_params_kernel<d><<<grid, FinCfg<d>::T, 0, stream>>>(d_stats, d_avgvar, t->d_shift_f, t->d_scale, d_set, t->Kmax, K, kp, \
                                                                     t->d_bimg, t->d_ck, d_ll, d_bad, iter, fault_iter)
    switch (t->D) {
        case 8: GMM_FIN(8); break;
        case 16: GMM_FIN(16); break;
        case 24: GMM_FIN(24); break;
        default: return fail(GMM_ERR_ARG, "device-side finalisation: unsupported D");
    }
#undef GMM_FIN
    CUDA_TRY(cudaGetLastError());
    t->e_NG = (K + 15) / 16;
    return GMM_OK;
}

template <int D>
static int launch_estep_d(TcState* t, int K, const float* x, int n, float* memb, size_t pitch, float* den, double* d_ll, const float* w,
                          cudaStream_t stream) {
    using C = ECfg<D>;
    using L = EsCfg<D>;
    // one instance per number of resident supergroups (1 .. 4) of a pass, unweighted and weighted
    using KernFn = void (*)(const float*, const uint8_t*, const float*, const float*, const float*, float*, size_t, int, int, double*, int,
                            const float*, float*, const float*);
    static const KernFn kern0[C::MAXSG] = {estep_tc_kernel<D, 1>, estep_tc_kernel<D, 2>, estep_tc_kernel<D, 3>, estep_tc_kernel<D, 4>};
    static const KernFn kern1[C::MAXSG] = {estep_tc_kernel<D, 1, true>, estep_tc_kernel<D, 2, true>, estep_tc_kernel<D, 3, true>,
                                           estep_tc_kernel<D, 4, true>};
    static_assert(C::MAXSG == 4, "one kernel instance per supergroup count");
    if (!t->attr_estep) {
        for (auto* k : kern0) CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, L::SMEM_BYTES));
        for (auto* k : kern1) CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, L::SMEM_BYTES));
        t->attr_estep = true;
    }
    const KernFn* kern = w ? kern1 : kern0;
    const int ntiles = (n + 127) / 128;
    int grid = t->num_sms;
    if (grid > ntiles) grid = ntiles;
    if (grid < 1) grid = 1;
    const int NP = (K + 63) / 64;
    if (NP > 1 && !den) return fail(GMM_ERR_STATE, "tensor E-step: context was created for at most 64 clusters");
    // P passes of 64 clusters: log-denominators of passes 0 .. P-2 (mode 1), then the last pass writes its final
    // responsibilities and the events' total log-denominators (mode 2, or mode 0 when P = 1), then passes 0 .. P-2 write
    // theirs against those totals (mode 3): 2P - 1 launches, every responsibility stored once
    auto launch = [&](int p, int mode, const float* den_in, float* den_out) {
        const int Kp = K - 64 * p < 64 ? K - 64 * p : 64;
        kern[(Kp + C::GB - 1) / C::GB - 1]<<<grid, L::THREADS, L::SMEM_BYTES, stream>>>(
            x, t->d_bimg + (size_t)p * C::MAXSG * C::B_SG, t->d_ck + 128 * p, t->d_shift_f, t->d_inv_scale_f,
            memb + (size_t)(64 * p) * pitch, pitch, n, Kp, d_ll, mode, den_in, den_out, w);
        return cudaGetLastError();
    };
    if (NP == 1) CUDA_TRY(launch(0, 0, nullptr, nullptr));
    else {
        for (int p = 0; p + 1 < NP; p++) CUDA_TRY(launch(p, 1, p ? den : nullptr, den));
        CUDA_TRY(launch(NP - 1, 2, den, den));
        for (int p = 0; p + 1 < NP; p++) CUDA_TRY(launch(p, 3, den, nullptr));
    }
    return GMM_OK;
}

static int launch_estep_any(TcState* t, int K, const float* x, int n, float* memb, size_t pitch, float* den, double* d_ll, const float* w,
                            cudaStream_t stream) {
    if (!t || !t->emap_ok) return fail(GMM_ERR_STATE, "tensor E-step not initialised for this shape");
    switch (t->D) {
        case 8: return launch_estep_d<8>(t, K, x, n, memb, pitch, den, d_ll, w, stream);
        case 16: return launch_estep_d<16>(t, K, x, n, memb, pitch, den, d_ll, w, stream);
        case 24: return launch_estep_d<24>(t, K, x, n, memb, pitch, den, d_ll, w, stream);
        default: return fail(GMM_ERR_ARG, "tensor E-step: unsupported D");
    }
}

int tc_launch_estep(TcState* t, int K, double* d_ll, cudaStream_t stream, const float* d_w) {
    if (!t) return fail(GMM_ERR_STATE, "tensor E-step not initialised for this shape");
    return launch_estep_any(t, K, t->d_x, t->n, t->d_memb, t->memb_pitch, t->d_den, d_ll, d_w, stream);
}

int tc_launch_estep_on(TcState* t, int K, const float* d_x_aos, int n, float* d_memb, size_t pitch, float* d_den, double* d_ll,
                       cudaStream_t stream) {
    if (n <= 0) return GMM_OK;
    return launch_estep_any(t, K, d_x_aos, n, d_memb, pitch, d_den, d_ll, nullptr, stream);
}

template <int D>
static int launch_score_d(TcState* t, int K, const TcScoreIo& io, cudaStream_t stream) {
    using C = ECfg<D>;
    static void (*const kern[C::MAXSG])(const float*, const uint8_t*, const float*, const float*, const float*, int, int, int, int, int,
                                        float*, float*, int*, int*, float*, float*, double*, int*) = {
        score_tc_kernel<D, 1>, score_tc_kernel<D, 2>, score_tc_kernel<D, 3>, score_tc_kernel<D, 4>};
    static_assert(C::MAXSG == 4, "one kernel instance per supergroup count");
    if (!t->attr_score) {
        for (auto* k : kern) CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
        t->attr_score = true;
    }
    const int ntiles = (io.n + 127) / 128;
    int grid = t->num_sms;
    if (grid > ntiles) grid = ntiles;
    if (grid < 1) grid = 1;
    const int NP = (K + 63) / 64;
    if (NP > 1 && !(io.run_den && io.run_bl && io.run_bk)) return fail(GMM_ERR_STATE, "tensor scoring: no running state for K > 64");
    for (int p = 0; p < NP; p++) {
        const int Kp = K - 64 * p < 64 ? K - 64 * p : 64;
        kern[(Kp + C::GB - 1) / C::GB - 1]<<<grid, C::THREADS, C::SMEM_BYTES, stream>>>(
            io.x, t->d_bimg + (size_t)p * C::MAXSG * C::B_SG, t->d_ck + 128 * p, t->d_shift_f, t->d_inv_scale_f, io.n, Kp, 64 * p, p, p + 1 == NP, io.run_den, io.run_bl, io.run_bk, io.labels, io.max_resp, io.logp, io.ll,
            io.flag);
        CUDA_TRY(cudaGetLastError());
    }
    return GMM_OK;
}

int tc_launch_score(TcState* t, int K, const TcScoreIo& io, cudaStream_t stream) {
    if (!t || !t->emap_ok) return fail(GMM_ERR_STATE, "tensor scoring not initialised for this shape");
    if (io.n <= 0) return GMM_OK;
    switch (t->D) {
        case 8: return launch_score_d<8>(t, K, io, stream);
        case 16: return launch_score_d<16>(t, K, io, stream);
        case 24: return launch_score_d<24>(t, K, io, stream);
        default: return fail(GMM_ERR_ARG, "tensor scoring: unsupported D");
    }
}

// K <= 32: one CTA per event range and 32 clusters.  K > 32: two CTAs per range and 64 clusters, each building half of the
// feature rows (MCfg): the feature operand is built once per 64 clusters, and both CTAs read the range's tiles in one wave.
template <int D>
static int launch_mstep_d(TcState* t, int K, const CUtensorMap& tm_x, const CUtensorMap& tm_g, int n, double* d_stats, const float* w,
                          double wscale, cudaStream_t stream) {
    using C32 = MCfg<D, 32>;
    using C64 = MCfg<D, 64>;
    static_assert(C32::SMEM_BYTES <= 232448 && C64::SMEM_BYTES <= 232448, "shared memory budget");
    if (!t->attr_mstep) {
        CUDA_TRY(cudaFuncSetAttribute(mstep_tc_kernel<D, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, C32::SMEM_BYTES));
        CUDA_TRY(cudaFuncSetAttribute(mstep_tc_kernel<D, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, C64::SMEM_BYTES));
        CUDA_TRY(cudaFuncSetAttribute(mstep_tc_kernel<D, 32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, C32::SMEM_BYTES));
        CUDA_TRY(cudaFuncSetAttribute(mstep_tc_kernel<D, 64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, C64::SMEM_BYTES));
        t->attr_mstep = true;
    }
    const float w_max = (float)wscale, w_inv = (float)(1.0 / wscale);
    int gx = t->num_sms;
    int per = (n + gx - 1) / gx;
    per = (per + kTE - 1) / kTE * kTE;
    gx = (n + per - 1) / per;
    const bool pair = K > 32;
    const int ncl = pair ? 64 : 32;
    const int gy = (K + ncl - 1) / ncl;
    if ((size_t)gx * gy * (ncl / kNCL) * C32::MT * 128 * kNCL > t->d_scratch.size()) return fail(GMM_ERR_STATE, "tensor M-step scratch too small");
    const dim3 grid(pair ? 2 * gx : gx, gy);
    if (pair) {
        if (w) mstep_tc_kernel<D, 64, true><<<grid, C64::THREADS, C64::SMEM_BYTES, stream>>>(tm_x, tm_g, n, K, t->d_scratch, per, t->magic, t->d_opmap, w, w_max, w_inv);
        else mstep_tc_kernel<D, 64><<<grid, C64::THREADS, C64::SMEM_BYTES, stream>>>(tm_x, tm_g, n, K, t->d_scratch, per, t->magic, t->d_opmap, nullptr, 1.0f, 1.0f);
    } else {
        if (w) mstep_tc_kernel<D, 32, true><<<grid, C32::THREADS, C32::SMEM_BYTES, stream>>>(tm_x, tm_g, n, K, t->d_scratch, per, t->magic, t->d_opmap, w, w_max, w_inv);
        else mstep_tc_kernel<D, 32><<<grid, C32::THREADS, C32::SMEM_BYTES, stream>>>(tm_x, tm_g, n, K, t->d_scratch, per, t->magic, t->d_opmap, nullptr, 1.0f, 1.0f);
    }
    CUDA_TRY(cudaGetLastError());
    mstep_tc_finalize_kernel<<<C32::MT * 128, 256, 0, stream>>>(t->d_scratch, gx, C32::MT, K, C32::F, t->d_rowmap, t->d_scale, d_stats,
                                                                w ? wscale : 1.0);
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

static int launch_mstep_any(TcState* t, int K, const CUtensorMap& tm_x, const CUtensorMap& tm_g, int n, double* d_stats, const float* w,
                            double wscale, cudaStream_t stream) {
    if (!t || !t->maps_ok) return fail(GMM_ERR_STATE, "tensor-core M-step not initialised for this shape");
    if (!t->have_shift) return fail(GMM_ERR_STATE, "tensor-core M-step needs gmm_seed (shift/scale) first");
    if (!t->mstep_ready) return fail(GMM_ERR_STATE, "tensor-core M-step: the data range exceeds the fixed-point operand budget");
    switch (t->D) {
        case 4: return launch_mstep_d<4>(t, K, tm_x, tm_g, n, d_stats, w, wscale, stream);
        case 8: return launch_mstep_d<8>(t, K, tm_x, tm_g, n, d_stats, w, wscale, stream);
        case 12: return launch_mstep_d<12>(t, K, tm_x, tm_g, n, d_stats, w, wscale, stream);
        case 16: return launch_mstep_d<16>(t, K, tm_x, tm_g, n, d_stats, w, wscale, stream);
        case 20: return launch_mstep_d<20>(t, K, tm_x, tm_g, n, d_stats, w, wscale, stream);
        case 24: return launch_mstep_d<24>(t, K, tm_x, tm_g, n, d_stats, w, wscale, stream);
        default: return fail(GMM_ERR_ARG, "tensor-core M-step: unsupported D");
    }
}

int tc_launch_mstep(TcState* t, int K, double* d_stats, cudaStream_t stream, const float* d_w, double wscale) {
    if (!t) return fail(GMM_ERR_STATE, "tensor-core M-step not initialised for this shape");
    return launch_mstep_any(t, K, t->tm_x, t->tm_g, t->n, d_stats, d_w, wscale, stream);
}

int tc_launch_mstep_on(TcState* t, int K, const float* d_z, const float* d_memb, size_t pitch, int n, double* d_stats, cudaStream_t stream) {
    if (n <= 0) return GMM_OK;
    if (!t || !t->maps_ok) return fail(GMM_ERR_STATE, "tensor-core M-step not initialised for this shape");
    if (t->cmap_z != d_z || t->cmap_g != d_memb || t->cmap_pitch != pitch || t->cmap_n != n) {
        t->cmap_n = -1;
        if (int rc = make_map_2d(&t->tm_cx, d_z, (uint64_t)n, (uint64_t)t->D, (uint64_t)pitch * 4, kTE, (uint32_t)t->D, /*swizzle128=*/true)) return rc;
        if (int rc = make_map_2d(&t->tm_cg, d_memb, (uint64_t)n, (uint64_t)t->Kmax, (uint64_t)pitch * 4, kTE, kNCL, /*swizzle128=*/true)) return rc;
        t->cmap_z = d_z; t->cmap_g = d_memb; t->cmap_pitch = pitch; t->cmap_n = n;
    }
    return launch_mstep_any(t, K, t->tm_cx, t->tm_cg, n, d_stats, nullptr, 1.0, stream);
}

const float* tc_shift_f(const TcState* t) { return t && t->have_shift ? t->d_shift_f.get() : nullptr; }
const float* tc_inv_scale_f(const TcState* t) { return t && t->have_shift ? t->d_inv_scale_f.get() : nullptr; }
float tc_mstep_zbound(const TcState* t) {
    float zb = 0.f;
    if (t)
        for (int d = 0; d < t->D; d++) zb = std::fmax(zb, t->zmax[d]);
    return zb;
}

}  // namespace gmm
