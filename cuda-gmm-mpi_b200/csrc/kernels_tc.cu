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
// With B = [gh ; gl] stacked as ONE N = 64 operand, ph x [gh ; gl] is a single MMA that fills both column groups;
// pl x gs (N = 32) adds into the second group.
//
// Dataflow per CTA (persistent over a contiguous range of events, 32 clusters per CTA row of the grid):
//   warp 0      TMA producer: tile [D][32 events] of the pre-standardised SoA copy z and raw
//               responsibility tile [32 clusters][32 events] (2-D tensor maps, SWIZZLE_128B for
//               the latter, zero fill out of bounds)
//   warps 4-11  operand builders (two warpgroups on alternate tiles): form the products, split
//               them, write the wgmma operand images (no-swizzle core-matrix layout)
//   warpgroups 3 .. 2+MT  consumers, one per 128-row feature tile: per 32 events 2 x 2 x (m64n64k16 + m64n32k16)
//               wgmma with the accumulators in registers.  The exact group is drained every 128 events and the
//               remainder group every 512 into FP32 round-to-nearest partial sums held in shared memory (one private
//               slot per thread), written ONCE per CTA (no scratch zeroing, no atomics).
// A second tiny kernel reduces the per-CTA partials in double and un-scales.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#if defined(__F16C__) && defined(__AVX__)
#include <immintrin.h>
#endif
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_math.h"
#include "kernels_tc.cuh"
#include "tc_ptx.cuh"

namespace gmm {

using namespace ptx;

#define TC_CUDA_TRY(expr)                                                                     \
    do {                                                                                      \
        cudaError_t e_ = (expr);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return fail(GMM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));    \
    } while (0)

// ---------------------------------------------------------------------------
// M-step kernel configuration
// ---------------------------------------------------------------------------
constexpr int kTE = 32;          // events per sub-tile (MMA K extent per operand part)
constexpr int kNCL = 32;         // clusters per CTA pass (N of the exact / remainder groups: register budget of the consumers)
constexpr int kNST = 2;          // operand stages
constexpr int kNRAW = 4;         // raw (TMA) stages
constexpr int kChunkSub = 4;     // sub-tiles per chain of the exact column group: 128 events (the bit budget below)
constexpr int kChunkSub2 = 16;   // sub-tiles per chain of the remainder column group (no exactness to protect: drained 4x less often)
// Bit budget of the exact accumulator: 11 (ph, every integer up to 2048 is an FP16 value) + 6 (gh) + 7 (128 events) = 24.
// The split favours phi: the remainder pl is rounded to FP16 RELATIVE to itself, so its (unbiased) rounding noise scales
// with the quantum of ph — on covariance entries 6e-6 per call with 9 + 8 bits, 1.2e-6 with 11 + 6 (scripts/emu_mstep.py).
constexpr int kPhiBits = 11;     // |ph| <= 2^11 quanta
constexpr float kGammaScale = 1024.0f;               // responsibilities are scaled by 2^10 in the operand
constexpr float kGammaMagic = 1.5f * 134217728.0f;   // 1.5 * 2^27: ulp = 16 = 2^-6 in the scaled units

// Row layout of the feature operand.  The four warps of a builder warpgroup run ONE instruction stream (round 1 / early
// round 2 unrolled a different quarter of the feature list per warp: 50 KB of SASS against a 32 KB L1.5 instruction cache,
// a third of the builders' stall samples were instruction fetch): warp p loads the event's coordinates ROTATED by p*D/4
// dimensions (a run-time shared-memory address) and evaluates the same canonical list of RPP rows on them —
//     r = 0                      1
//     r = 1 + a          (a < S) z'_a
//     r = 1 + S + a      (a < S) z'_a^2
//     r = 1 + 2S + a*D/2 + (d-1) (a < S, 1 <= d <= D/2)   z'_a * z'_{(a+d) mod D}
// with z'_t = z_{(t + pS) mod D}, S = D/4.  The rotations of the canonical pairs cover every unordered pair of
// dimensions once, except the D/2 antipodal pairs (d = D/2), which two warps produce (one copy is ignored), and the
// constant row (kept from warp 0).  Warp p writes operand rows [p*CPP*8, p*CPP*8 + RPP); tc_row_map() gives the packed
// statistic each row feeds.
template <int D> struct MCfg {
    static_assert(D % 4 == 0, "tensor M-step: D must be a multiple of 4");
    static constexpr int F = 1 + D + D * (D + 1) / 2;
    static constexpr int S = D / 4;                       // rotation step between the four builder warps
    static constexpr int RPP = 1 + 2 * S + S * (D / 2);   // canonical rows per warp
    static constexpr int CPP = (RPP + 7) / 8;             // 16-byte chunks per warp
    static constexpr int NCHUNK = 4 * CPP;                // chunks written per event
    static constexpr int MT = (NCHUNK * 8 + 127) / 128;   // M tiles of 128 feature rows
    static constexpr int PHI_PART = MT * 128 * kTE * 2;   // bytes of one part (leading or remainder)
    static constexpr int PHI_STAGE = 2 * PHI_PART;
    static constexpr int G_PART = kNCL * kTE * 2;
    static constexpr int G_STAGE = 3 * G_PART;            // [gh (64 rows) ; gl (64 rows)] = ONE K-major N = 128 image, then gs
    static constexpr int RAWX = D * kTE * 4;              // [D][32 events] from the SoA copy
    static constexpr int RAWG = kNCL * kTE * 4;
    static constexpr int OFF_PHI = 0;
    static constexpr int OFF_G = OFF_PHI + kNST * PHI_STAGE;
    static constexpr int OFF_RAWX = OFF_G + kNST * G_STAGE;
    static constexpr int OFF_RAWG = OFF_RAWX + kNRAW * RAWX;
    static constexpr int NCT = MT * 128;                  // consumer threads (one warpgroup per 128-row feature tile)
    static constexpr int OFF_RACC = OFF_RAWG + kNRAW * RAWG;   // [32][NCT] FP32 partial sums, one private column per thread
    static constexpr int OFF_BAR = OFF_RACC + 32 * NCT * 4;
    static constexpr int SMEM_BYTES = OFF_BAR + 512;
    static constexpr int THREADS = 384 + NCT;             // producer warpgroup, two builder warpgroups, consumers
    // register pools: producer / builders / consumers.  The kernel is launched with REG_LAUNCH registers per thread
    // (the __launch_bounds__ maximum, which ptxas uses when setmaxnreg is present); setmaxnreg only redistributes that
    // allocation, so a warpgroup's increase waits until the others' decreases have freed enough — the sum must fit.
    static constexpr int REG_LAUNCH = (65536 / THREADS) / 8 * 8 > 255 ? 255 : (65536 / THREADS) / 8 * 8;
    static constexpr int REG_P = MT == 1 ? 40 : 24;
    static constexpr int REG_B = MT == 3 ? 80 : 112;
    static constexpr int REG_C = MT == 3 ? 96 : (MT == 2 ? 112 : 240);
    static_assert(128 * REG_P + 256 * REG_B + NCT * REG_C <= THREADS * REG_LAUNCH, "register pools");
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

__host__ __device__ constexpr int tri_row(int t) {        // t = i(i+1)/2 + j, j <= i  ->  i
    int i = 0;
    while ((i + 1) * (i + 2) / 2 <= t) i++;
    return i;
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

// Leading part / remainder of canonical row r for the (rotated) event z (r is a compile-time constant after
// unrolling).  Products: both parts come from the EXACT product (fused multiply-adds), rounded once each.
template <int D>
__device__ __forceinline__ void feature_split(const float (&z)[D], int r, const MMagic& mg, float& h, float& l) {
    using C = MCfg<D>;
    if (r == 0) { h = 1.0f; l = 0.0f; }
    else if (r <= C::S) {
        const float v = z[r - 1];
        h = __fsub_rn(__fadd_rn(v, mg.lin), mg.lin);
        l = __fsub_rn(v, h);
    } else if (r < C::RPP) {
        int a, b;
        if (r <= 2 * C::S) { a = r - 1 - C::S; b = a; }
        else { const int t = r - 1 - 2 * C::S; a = t / (D / 2); b = (a + 1 + t % (D / 2)) % D; }
        h = __fsub_rn(__fmaf_rn(z[a], z[b], mg.prod), mg.prod);
        l = __fmaf_rn(z[a], z[b], -h);
    } else { h = 0.0f; l = 0.0f; }
}

// Builds the CPP 16-byte chunks of one event for builder warp `part` and stores both parts into the MN-major operand image:
//   byte(row, e) = (row/8)*512 + (e/8)*128 + (e%8)*16 + (row%8)*2        (LBO = 128, SBO = 512)
template <int D>
__device__ __forceinline__ void build_phi_chunks(const float (&z)[D], const MMagic& mg, uint8_t* hi_base, uint8_t* lo_base, int e, int part) {
    using C = MCfg<D>;
    const int eoff = part * (C::CPP * 512) + (e >> 3) * 128 + (e & 7) * 16;
#pragma unroll
    for (int c = 0; c < C::CPP; c++) {
        float hi[8], lo[8];
#pragma unroll
        for (int u = 0; u < 8; u++) feature_split<D>(z, c * 8 + u, mg, hi[u], lo[u]);
        uint4 h, l;
        h.x = pack_half2(hi[0], hi[1]); h.y = pack_half2(hi[2], hi[3]); h.z = pack_half2(hi[4], hi[5]); h.w = pack_half2(hi[6], hi[7]);   // exact: <= 2048 quanta
        l.x = pack_half2(lo[0], lo[1]); l.y = pack_half2(lo[2], lo[3]); l.z = pack_half2(lo[4], lo[5]); l.w = pack_half2(lo[6], lo[7]);
        *reinterpret_cast<uint4*>(hi_base + c * 512 + eoff) = h;
        *reinterpret_cast<uint4*>(lo_base + c * 512 + eoff) = l;
    }
}

// Packed statistic (index into a cluster's F values, -1 = ignored copy) and the two dimensions (-1 = none) behind
// operand row `row`; host side of the layout above.
struct RowInfo { int f, i, j; };
static RowInfo tc_row_info(int D, int row) {
    const int S = D / 4, RPP = 1 + 2 * S + S * (D / 2), CPP = (RPP + 7) / 8;
    const int p = row / (CPP * 8), r = row % (CPP * 8);
    RowInfo o{-1, -1, -1};
    if (p >= 4 || r >= RPP) return o;
    if (r == 0) { if (p == 0) o.f = 0; return o; }
    if (r <= S) { o.i = (r - 1 + p * S) % D; o.f = 1 + o.i; return o; }
    int a, b;
    if (r <= 2 * S) { a = r - 1 - S; b = a; }
    else { const int t = r - 1 - 2 * S; a = t / (D / 2); b = (a + 1 + t % (D / 2)) % D; }
    const int ta = (a + p * S) % D, tb = (b + p * S) % D;
    if (a != b && (b - a + D) % D == D / 2 && ta >= D / 2) return o;       // antipodal pair: the copy with the smaller first index counts
    o.i = ta > tb ? ta : tb;
    o.j = ta > tb ? tb : ta;
    o.f = feat2(D, o.i, o.j);
    return o;
}

// Feature tile `mt` is drained after sub-tile i when its 128-event chain ends there: the chains of the tiles are
// staggered by one sub-tile each, so that the consumer warpgroups do not all drain after the same sub-tile.
// The remainder column group rides along and is drained (and restarted) only at every fourth of those points.
__device__ __forceinline__ bool chain_ends(int i, int mt, int nsub) { return ((i + mt) % kChunkSub) == kChunkSub - 1 || i == nsub - 1; }
__device__ __forceinline__ bool chain_starts(int i, int mt) { return i == 0 || ((i + mt) % kChunkSub) == 0; }
__device__ __forceinline__ bool chain2_ends(int i, int mt, int nsub) { return ((i + mt) % kChunkSub2) == kChunkSub2 - 1 || i == nsub - 1; }
__device__ __forceinline__ bool chain2_starts(int i, int mt) { return i == 0 || ((i + mt) % kChunkSub2) == 0; }

template <int D>
__global__ void __launch_bounds__(MCfg<D>::THREADS, 1)
mstep_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_g, int n,
                float* __restrict__ scratch, int events_per_cta, const __grid_constant__ MMagic magic) {
    using C = MCfg<D>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
    uint64_t* raw_full = bars;                 // [kNRAW]
    uint64_t* raw_empty = bars + kNRAW;        // [kNRAW]
    uint64_t* op_full = bars + 2 * kNRAW;      // [kNST]
    uint64_t* op_empty = op_full + kNST;       // [kNST]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int e_begin = blockIdx.x * events_per_cta;
    const int e_end = min(n, e_begin + events_per_cta);
    const int nsub = (e_end - e_begin + kTE - 1) / kTE;
    const int k0 = blockIdx.y * kNCL;

    // ---- one-time setup ----
    for (int i = threadIdx.x * 16; i < C::OFF_RAWX; i += C::THREADS * 16) *reinterpret_cast<uint4*>(smem + i) = make_uint4(0, 0, 0, 0);
    if (threadIdx.x == 0) {
        for (int s = 0; s < kNRAW; s++) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], 4); }
        for (int s = 0; s < kNST; s++) { mbar_init(&op_full[s], 4); mbar_init(&op_empty[s], 4 * C::MT); }
        fence_mbar_init();
    }
    fence_proxy_async_smem();
    __syncthreads();

    if (warp < 4) {
        set_regs<C::REG_P, C::REG_LAUNCH>();
        if (warp == 0) {
            // ===================== TMA producer =====================
            if (elect_one()) {
                for (int i = 0; i < nsub; i++) {
                    const int st = i % kNRAW, ph = (i / kNRAW) & 1;
                    mbar_wait_parked(&raw_empty[st], ph ^ 1, 500);
                    mbar_arrive_expect_tx(&raw_full[st], kTE * D * 4 + C::RAWG);
                    const int e0 = e_begin + i * kTE;
                    tma_load_2d(smem + C::OFF_RAWX + st * C::RAWX, &tm_x, e0, 0, &raw_full[st]);
                    tma_load_2d(smem + C::OFF_RAWG + st * C::RAWG, &tm_g, e0, k0, &raw_full[st]);
                }
            }
        }
    } else if (warp < 12) {
        set_regs<C::REG_B, C::REG_LAUNCH>();
        // ===================== operand builders =====================
        // two builder warpgroups work on alternate sub-tiles (two sub-tiles in flight), the four warps
        // of a group split the 16-byte feature chunks (c = part mod 4)
        const int bwg = (warp - 4) >> 2;           // sub-tiles i = bwg (mod 2)
        const int part = (warp - 4) & 3;
        const int bt = threadIdx.x - 128 - bwg * 128;   // 0..127 inside the group
        for (int i = bwg; i < nsub; i += 2) {
            const int rs = i % kNRAW, rph = (i / kNRAW) & 1;
            const int os = i % kNST, oph = (i / kNST) & 1;
            mbar_wait_parked(&raw_full[rs], rph, 200);
            // --- features of event `lane` ---
            float z[D];                                // already centred and scaled (tc_set_shift_scale writes the z copy), rotated by part * S
            {
                const float* xr = reinterpret_cast<const float*>(smem + C::OFF_RAWX + rs * C::RAWX) + lane;   // [d][32]: conflict-free
                int dd = part * C::S;
#pragma unroll
                for (int d = 0; d < D; d++) { z[d] = xr[dd * kTE]; dd = dd + 1 == D ? 0 : dd + 1; }
            }
            // --- responsibilities: thread -> (cluster row k, 8-event chunk ce), one item per thread.
            // The raw tile is written by TMA with SWIZZLE_128B (16-byte chunk c of row r sits at chunk
            // c ^ (r & 7)), so 8 lanes reading the same chunk of 8 consecutive rows hit 8 different
            // bank groups; the operand image puts the 4 K-chunks of an 8-row group next to each other
            // (LBO = 128, SBO = 512), so a warp stores 512 contiguous bytes: no bank conflicts either way.
            uint4 gh, gl, gs;
            float gdep;
            {
                const int kg = bt >> 5, l = bt & 31;
                const int k = kg * 8 + (l & 7), ce = l >> 3;
                const uint8_t* grow = smem + C::OFF_RAWG + rs * C::RAWG + k * (kTE * 4);
                const float4 a = *reinterpret_cast<const float4*>(grow + (((2 * ce) ^ (k & 7)) << 4));
                const float4 b = *reinterpret_cast<const float4*>(grow + (((2 * ce + 1) ^ (k & 7)) << 4));
                const float g[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                gdep = a.x + b.x;
                float hi[8], lo[8];
#pragma unroll
                for (int u = 0; u < 8; u++) {                  // gh = 16 * round(64 g) (0 .. 1024), gl = 1024 g - gh, both from the exact product
                    hi[u] = __fsub_rn(__fmaf_rn(g[u], kGammaScale, kGammaMagic), kGammaMagic);
                    lo[u] = __fmaf_rn(g[u], kGammaScale, -hi[u]);
                }
                gh = make_uint4(pack_half2(hi[0], hi[1]), pack_half2(hi[2], hi[3]), pack_half2(hi[4], hi[5]), pack_half2(hi[6], hi[7]));
                gl = make_uint4(pack_half2(lo[0], lo[1]), pack_half2(lo[2], lo[3]), pack_half2(lo[4], lo[5]), pack_half2(lo[6], lo[7]));
                gs = make_uint4(pack_half2(g[0] * kGammaScale, g[1] * kGammaScale), pack_half2(g[2] * kGammaScale, g[3] * kGammaScale),
                                pack_half2(g[4] * kGammaScale, g[5] * kGammaScale), pack_half2(g[6] * kGammaScale, g[7] * kGammaScale));
            }
            // The raw tiles must BE in registers before the stage goes back to the TMA producer: an mbarrier arrive does
            // not wait for the warp's outstanding shared-memory loads.  The arrive is therefore made data-dependent on
            // every load of this thread: a sum over z and one component of the responsibility vector, folded into the
            // arrive's own operand list below (the asm statement consumes the value, so neither the compiler nor the
            // hardware can retire it before the loads have landed).
            float dep = gdep;
#pragma unroll
            for (int d = 0; d < D; d++) dep += z[d];
            __syncwarp();
            if (lane == 0) mbar_arrive_after(&raw_empty[rs], dep);
            else asm volatile("" ::"f"(dep));
            mbar_wait_parked(&op_empty[os], oph ^ 1, 200);
            uint8_t* phi_hi = smem + C::OFF_PHI + os * C::PHI_STAGE;
            uint8_t* phi_lo = phi_hi + C::PHI_PART;
            build_phi_chunks<D>(z, magic, phi_hi, phi_lo, lane, part);
            {
                // K-major B image: byte(k, e) = (k/8)*512 + (e/8)*128 + (k%8)*16 + (e%8)*2      (LBO = 128, SBO = 512); gl = rows 32..63
                uint8_t* g_hi = smem + C::OFF_G + os * C::G_STAGE;
                const int kg = bt >> 5, l = bt & 31;
                *reinterpret_cast<uint4*>(g_hi + kg * 512 + l * 16) = gh;
                *reinterpret_cast<uint4*>(g_hi + C::G_PART + kg * 512 + l * 16) = gl;
                *reinterpret_cast<uint4*>(g_hi + 2 * C::G_PART + kg * 512 + l * 16) = gs;
            }
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&op_full[os]);
        }
    } else {
        set_regs<C::REG_C, C::REG_LAUNCH>();
        // ===================== consumers: wgmma, accumulators in registers =====================
        const int mt = (warp - 12) >> 2;                           // feature tile of this warpgroup (rows 128 mt ..)
        const int ct = threadIdx.x - 384;                          // consumer thread 0 .. NCT-1
        const int wq = warp & 3, gid = lane >> 2, qd = lane & 3;
        float* racc = reinterpret_cast<float*>(smem + C::OFF_RACC) + ct;     // [32][NCT]: racc[j * NCT]
#pragma unroll
        for (int j = 0; j < 32; j++) racc[j * C::NCT] = 0.0f;
        float acc[2][32];                                          // per 64-row half: regs 0-15 exact group, 16-31 remainder group
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int j = 0; j < 32; j++) acc[h][j] = 0.0f;
        for (int i = 0; i < nsub; i++) {
            const int os = i % kNST, oph = (i / kNST) & 1;
            mbar_wait_parked(&op_full[os], oph, 100);
            const uint32_t phi = smem_u32(smem + C::OFF_PHI + os * C::PHI_STAGE);
            const uint32_t gam = smem_u32(smem + C::OFF_G + os * C::G_STAGE);
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; h++) {
#pragma unroll
                for (int ks = 0; ks < kTE / 16; ks++) {
                    const uint64_t bdesc = make_smem_desc(gam + ks * 256, /*LBO*/ 128, /*SBO*/ 512);     // rows 0-31 gh, 32-63 gl
                    const uint64_t sdesc = make_smem_desc(gam + 2 * C::G_PART + ks * 256, 128, 512);     // gs
                    const uint32_t arow = mt * 8192 + h * 4096 + ks * 256;
                    const uint64_t ah = make_smem_desc(phi + arow, /*LBO*/ 128, /*SBO*/ 512);
                    const uint64_t al = make_smem_desc(phi + C::PHI_PART + arow, 128, 512);
                    wgmma_m64n64k16_ss_tn(acc[h], ah, bdesc);                                          // [ph gh | ph gl]
                    wgmma_m64n32k16_ss_tn(*reinterpret_cast<float(*)[16]>(&acc[h][16]), al, sdesc);     //        += pl gs
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&op_empty[os]);         // operand stage reusable: these MMAs have read it
            // drain: exact group at the end of its 128-event chain, remainder group at the end of its longer chain
            if (chain_ends(i, mt, nsub)) {
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int j = 0; j < 16; j++) { racc[(h * 16 + j) * C::NCT] += acc[h][j]; acc[h][j] = 0.0f; }
            }
            if (chain2_ends(i, mt, nsub)) {
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int j = 0; j < 16; j++) { racc[(h * 16 + j) * C::NCT] += acc[h][16 + j]; acc[h][16 + j] = 0.0f; }
            }
        }
        // one plain store of this thread's partial sums: [cta][tile][row][32 clusters]
        float* my = scratch + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * C::MT * 128 * kNCL + (size_t)mt * 128 * kNCL;
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int j = 0; j < 16; j += 2) {
                const int row = h * 64 + wq * 16 + gid + 8 * ((j >> 1) & 1);
                const int col = (j >> 2) * 8 + 2 * qd;
                *reinterpret_cast<float2*>(my + (size_t)row * kNCL + col) =
                    make_float2(racc[(h * 16 + j) * C::NCT], racc[(h * 16 + j + 1) * C::NCT]);
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
__global__ void __launch_bounds__(256)
mstep_tc_finalize_kernel(const float* __restrict__ scratch, int ncta_x, int MT, int K, int F, const int3* __restrict__ rowmap,
                         const double* __restrict__ scale, double* __restrict__ stats) {
    // one block per operand row; thread -> (cluster column, eighth of the CTAs): 128-byte coalesced reads
    constexpr int NQ = 256 / kNCL;
    __shared__ double part[NQ][kNCL];
    const int3 rm = rowmap[blockIdx.x];
    if (rm.x < 0) return;
    const int mt = blockIdx.x / 128, row = blockIdx.x % 128;
    const int col = threadIdx.x & (kNCL - 1), q = threadIdx.x / kNCL;
    double fac = 1.0 / (double)kGammaScale;
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
// One persistent CTA per SM, NWG independent warpgroups; each takes 64-event tiles in turn and per supergroup of 16
// clusters and block c of 8 output dimensions issues the k-steps that block needs (m64n128k16, A from registers),
// then squares and sums the 8 columns of each cluster (a quad of lanes holds them), the log-sum-exp over the
// clusters (again within the quad) and writes the responsibilities and the log-likelihood.  The warpgroups
// interleave, so one's MMAs overlap another's epilogue.
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
    static constexpr int NWG = 2;                             // warpgroups per CTA (255 registers each: no spills at D = 24)
    static constexpr int THREADS = 128 * NWG;
};

template <int D>
__global__ void __launch_bounds__(ECfg<D>::THREADS, 1)
estep_tc_kernel(const float* __restrict__ x_aos, const uint8_t* __restrict__ b_img, const float* __restrict__ ck,
                const float* __restrict__ shift_f, const float* __restrict__ inv_scale_f, float* __restrict__ memb,
                size_t pitch, int n, int K, int NSG, double* __restrict__ ll_out, int mode, const float* den_in,
                float* den_out) {
    // K / NSG / b_img / ck / memb describe ONE pass of at most 64 clusters.  More than 64 clusters take 2P - 1 launches
    // for P passes, and every responsibility is written exactly once:
    //   mode 1 (passes 0 .. P-2)  log-denominator only: den_out[e] = ln(sum_k exp(logit)) (+ den_in[e] in log space), no stores
    //   mode 2 (pass P-1)         its own log-sum-exp joined with den_in[e] (all other passes): final responsibilities of this
    //                             pass, den_out[e] = the event's total log-denominator, log-likelihood
    //   mode 3 (passes 0 .. P-2)  responsibilities against the known total den_in[e]: no log-sum-exp
    //   mode 0                    single pass (K <= 64)
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

    if (threadIdx.x == 0) { mbar_init(b_full, 1); fence_mbar_init(); }
    // base-2 logits in the epilogue: l2 = ck * log2(e) + (-0.5 * log2(e) / scale_k^2) * |scale_k * y|^2   (the per-cluster
    // power-of-two scale_k keeps the FP16 whitening factors in range whatever the cluster's width, see bimg_cluster)
    if (threadIdx.x < 64) { ck_s[threadIdx.x] = ck[threadIdx.x] * 1.4426950408889634f; ck_s[64 + threadIdx.x] = ck[64 + threadIdx.x]; }
    if (threadIdx.x < D) { sh_s[threadIdx.x] = shift_f[threadIdx.x]; isc_s[threadIdx.x] = inv_scale_f[threadIdx.x]; }
    __syncthreads();
    if (threadIdx.x == 0) {                    // resident B operand: one TMA bulk copy per block
        mbar_arrive_expect_tx(b_full, (uint32_t)NSG * C::B_SG);
        for (int g = 0; g < NSG * CP; g++) tma_load_1d(smem + C::OFF_B + g * C::B_BLOCK, b_img + (size_t)g * C::B_BLOCK, C::B_BLOCK, b_full);
    }

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
    constexpr uint32_t CH = C::N * 16;                        // bytes per B chunk
    double ll_acc = 0.0;
    constexpr float kLn2 = 0.6931471805599453f;
    mbar_wait(b_full, 0);

    for (; t < ntiles; t += stride) {
        uint32_t zh[CP][2], zl[CP][2];                         // [chunk][row]: FP16 pairs, hi and lo parts
#pragma unroll
        for (int j = 0; j < CP; j++) {
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
        const long long e0 = (long long)t * 64 + r0, e1 = e0 + 8;
        if (t + stride < ntiles) load_rows(t + stride);

        float lg[C::MAXSG][8];                                 // base-2 logits: [supergroup][4 clusters x 2 rows]
#pragma unroll
        for (int sg = 0; sg < C::MAXSG; sg++) {
            if (sg >= NSG) {
#pragma unroll
                for (int u = 0; u < 8; u++) lg[sg][u] = -INFINITY;
                continue;
            }
            float sq[32];                                      // sums of squares: [cluster 0..15][row]
#pragma unroll
            for (int u = 0; u < 32; u++) sq[u] = 0.f;
#pragma unroll
            for (int c = 0; c < CP; c++) {
                const uint32_t bb = bsm + (uint32_t)(sg * CP + c) * C::B_BLOCK;
                float acc[64];
#pragma unroll
                for (int u = 0; u < 64; u++) acc[u] = 0.f;
                wgmma_fence();
                bool accum = false;
#pragma unroll
                for (int j = c; j < CP; j++) {                 // (Wh_j, Wl_j) x (zh_j, zh_j)
                    wgmma_m64n128k16_rs(acc, zh[j][0], zh[j][1], zh[j][0], zh[j][1], make_smem_desc(bb + j * CH, CP * CH, 128), accum);
                    accum = true;
                }
                // (Wh_j) x (zl_j) for j >= c, then v x ones, two at a time; a lone v step pairs with a zero A chunk
#pragma unroll
                for (int p = c; p < CP + 1; p += 2) {
                    const int x = p, y = p + 1;                // list items: j < CP -> Wh_j x zl_j, j == CP -> v x ones
                    if (y <= CP) {
                        const uint32_t yc = y < CP ? (uint32_t)y : 2u * CP;
                        const uint32_t a2 = y < CP ? zl[y < CP ? y : 0][0] : ones, a3 = y < CP ? zl[y < CP ? y : 0][1] : ones;
                        wgmma_m64n128k16_rs(acc, zl[x][0], zl[x][1], a2, a3, make_smem_desc(bb + x * CH, (yc - x) * CH, 128), true);
                    } else {                                   // x == CP: v alone, paired with chunk c under a zero A chunk
                        wgmma_m64n128k16_rs(acc, 0u, 0u, ones, ones, make_smem_desc(bb + c * CH, (2 * CP - c) * CH, 128), true);
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    sq[2 * i] = fmaf(acc[4 * i], acc[4 * i], fmaf(acc[4 * i + 1], acc[4 * i + 1], sq[2 * i]));
                    sq[2 * i + 1] = fmaf(acc[4 * i + 2], acc[4 * i + 2], fmaf(acc[4 * i + 3], acc[4 * i + 3], sq[2 * i + 1]));
                }
            }
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
        // log-sum-exp over the clusters (estep2, gaussian_kernel.cu:481-503), per row: this lane's 16 logits, then the quad
        float mx[2] = {-INFINITY, -INFINITY};
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
                        const float g = fmaxf(denom, dx[r]);
                        const float tot = g + logf(__expf(denom - g) + __expf(dx[r] - g));
                        scale[r] *= __expf(denom - tot);
                        denom = tot;
                    }
                    if (qd == 0) den_out[er[r]] = denom;
                }
                if (qd == 0 && er[r] < n && (mode == 0 || mode == 2)) ll_acc += (double)denom;
            }
        }
        if (mode != 1) {
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

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
struct TcState {
    const float* d_x = nullptr;
    const float* d_x_soa = nullptr;
    float* d_z_soa = nullptr;        // [D][memb_pitch] centred/scaled SoA copy (M-step TMA source)
    float* d_memb = nullptr;
    size_t memb_pitch = 0;
    int n = 0, D = 0, Kmax = 0, num_sms = 132;
    CUtensorMap tm_x{}, tm_g{};
    bool maps_ok = false;
    float* d_shift_f = nullptr;      // [32]
    float* d_inv_scale_f = nullptr;  // [32]
    double* d_scale = nullptr;       // [32] = 1 / inv_scale_f (double)
    float* d_scratch = nullptr;      // [CTAs][MT][128][64] per-CTA partial sums, written once per launch
    size_t scratch_floats = 0;
    bool have_shift = false;
    bool mstep_ready = false;        // the fixed-point quanta of the feature rows are set and inside the supported range
    float zmax[GMM_MAX_DIMENSIONS] = {0};    // power-of-two bound of |z_d| over the whole data set
    MMagic magic{0.f, 0.f};          // rounding constants of the coordinate / product rows
    int3* d_rowmap = nullptr;        // [MT * 128] operand row -> (packed statistic, dimension i, dimension j)
    // E-step
    CUtensorMap tm_x128{};
    bool emap_ok = false;
    uint8_t* d_bimg = nullptr;       // [MAXNG * B_GROUP] resident B operand image
    uint8_t* h_bimg = nullptr;       // pinned
    size_t bimg_bytes = 0;
    uint8_t* d_opnd = nullptr;       // [ck (e_ck_len floats) | B image]; d_ck / d_bimg point into it
    uint8_t* h_opnd = nullptr;       // pinned mirror
    cudaEvent_t ev_h2d = nullptr;    // the last operand copy has left the pinned buffer
    bool h2d_pending = false;
    float* d_ck = nullptr;           // [passes][ck 64 | mult 64]: additive constant and quadratic-form multiplier per cluster
    float* h_ck = nullptr;           // pinned mirror
    float* d_den = nullptr;          // [memb_pitch] running / total log-denominator per event (Kmax > 64 only)
    int e_ck_len = 0;                // Kmax rounded up to whole passes of 64
    int e_NG = 0;
    int host_threads = 8;
    // cudaFuncAttributeMaxDynamicSharedMemorySize is per device: the "already set" flags live with the (per-device) state
    bool attr_estep = false, attr_mstep = false;
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
    TC_CUDA_TRY(cudaMalloc(&t->d_shift_f, sizeof(float) * GMM_MAX_DIMENSIONS));
    TC_CUDA_TRY(cudaMalloc(&t->d_inv_scale_f, sizeof(float) * GMM_MAX_DIMENSIONS));
    TC_CUDA_TRY(cudaMalloc(&t->d_scale, sizeof(double) * GMM_MAX_DIMENSIONS));
    // tensor maps: SoA events [D][pitch] viewed as (events, dims) -> smem tile [D][32 events];
    // responsibilities [Kmax][pitch] viewed as (events, clusters)
    TC_CUDA_TRY(cudaMalloc(&t->d_z_soa, sizeof(float) * memb_pitch * D));
    if (int rc = make_map_2d(&t->tm_x, t->d_z_soa, (uint64_t)n, (uint64_t)D, (uint64_t)memb_pitch * 4, kTE, (uint32_t)D)) return rc;
    if (int rc = make_map_2d(&t->tm_g, d_memb, (uint64_t)n, (uint64_t)Kmax, (uint64_t)memb_pitch * 4, kTE, kNCL, /*swizzle128=*/true)) return rc;
    t->maps_ok = true;
    if (D == 8 || D == 16 || D == 24) {
        const int passes = (Kmax + 63) / 64;
        t->e_ck_len = passes * 64;
        t->bimg_bytes = (size_t)passes * pass_bytes_for(D);
        // one staging / device buffer [ck | B image]: the operand of an iteration travels in ONE H2D copy
        const size_t ck_bytes = sizeof(float) * 2 * t->e_ck_len;     // 512 B per pass: keeps the image 16-byte aligned
        TC_CUDA_TRY(cudaMalloc(&t->d_opnd, ck_bytes + t->bimg_bytes));
        TC_CUDA_TRY(cudaMallocHost(&t->h_opnd, ck_bytes + t->bimg_bytes));
        t->d_ck = reinterpret_cast<float*>(t->d_opnd);
        t->h_ck = reinterpret_cast<float*>(t->h_opnd);
        t->d_bimg = t->d_opnd + ck_bytes;
        t->h_bimg = t->h_opnd + ck_bytes;
        TC_CUDA_TRY(cudaEventCreateWithFlags(&t->ev_h2d, cudaEventDisableTiming));
        if (passes > 1) TC_CUDA_TRY(cudaMalloc(&t->d_den, sizeof(float) * memb_pitch));
        t->emap_ok = true;
    }
    const int rpp = 1 + 2 * (D / 4) + (D / 4) * (D / 2), nrows = 4 * ((rpp + 7) / 8) * 8;
    const int mt = (nrows + 127) / 128;
    {
        std::vector<int3> rm((size_t)mt * 128);
        std::vector<char> seen((size_t)num_features(D), 0);
        for (int row = 0; row < mt * 128; row++) {
            const RowInfo ri = tc_row_info(D, row);
            rm[row] = make_int3(ri.f, ri.i, ri.j);
            if (ri.f >= 0) {
                if (seen[ri.f]) return fail(GMM_ERR_STATE, "tensor M-step row map: a statistic is produced twice");
                seen[ri.f] = 1;
            }
        }
        for (char c : seen) if (!c) return fail(GMM_ERR_STATE, "tensor M-step row map: a statistic is not produced");
        TC_CUDA_TRY(cudaMalloc(&t->d_rowmap, sizeof(int3) * rm.size()));
        TC_CUDA_TRY(cudaMemcpy(t->d_rowmap, rm.data(), sizeof(int3) * rm.size(), cudaMemcpyHostToDevice));
    }
    const int ytiles = (Kmax + kNCL - 1) / kNCL;
    t->scratch_floats = (size_t)num_sms * ytiles * mt * 128 * kNCL;
    TC_CUDA_TRY(cudaMalloc(&t->d_scratch, sizeof(float) * t->scratch_floats));
    return GMM_OK;
}

void tc_set_host_threads(TcState* t, int n) { if (t) t->host_threads = n < 1 ? 1 : n; }
bool tc_mstep_ready(const TcState* t) { return t && t->maps_ok && t->have_shift && t->mstep_ready; }
bool tc_estep_range_ok(const TcState* t) {
    if (!t || !t->have_shift) return false;
    for (int d = 0; d < t->D; d++)
        if (!(t->zmax[d] <= 16384.0f)) return false;
    return true;
}

void tc_destroy(TcState* t) {
    if (!t) return;
    cudaFree(t->d_shift_f); cudaFree(t->d_inv_scale_f); cudaFree(t->d_scale); cudaFree(t->d_scratch);
    cudaFree(t->d_opnd); cudaFree(t->d_den); cudaFree(t->d_z_soa); cudaFree(t->d_rowmap);
    if (t->h_opnd) cudaFreeHost(t->h_opnd);
    if (t->ev_h2d) cudaEventDestroy(t->ev_h2d);
    delete t;
}

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
    TC_CUDA_TRY(cudaMemcpyAsync(t->d_shift_f, sf, sizeof(sf), cudaMemcpyHostToDevice, stream));
    TC_CUDA_TRY(cudaMemcpyAsync(t->d_inv_scale_f, isf, sizeof(isf), cudaMemcpyHostToDevice, stream));
    TC_CUDA_TRY(cudaMemcpyAsync(t->d_scale, sc, sizeof(sc), cudaMemcpyHostToDevice, stream));
    {
        dim3 grid((unsigned)std::min<long long>(4LL * t->num_sms, ((long long)t->n + 255) / 256), (unsigned)t->D);
        standardise_soa_kernel<<<grid, 256, 0, stream>>>(t->d_x_soa, t->d_z_soa, t->memb_pitch, t->n, t->D, t->d_shift_f, t->d_inv_scale_f);
        TC_CUDA_TRY(cudaGetLastError());
    }
    TC_CUDA_TRY(cudaStreamSynchronize(stream));         // the staging arrays live on this stack frame
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
        TC_CUDA_TRY(cudaEventSynchronize(t->ev_h2d));
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
    TC_CUDA_TRY(cudaMemcpyAsync(t->d_opnd, t->h_opnd, sizeof(float) * 2 * t->e_ck_len + used, cudaMemcpyHostToDevice, stream));
    TC_CUDA_TRY(cudaEventRecord(t->ev_h2d, stream));
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
    __shared__ double sS[F + 3], sA[D][LD], sU[D][LD], sW[D][LD], sdm[D], sscale[D], svd[D], sredd[NW];
    __shared__ float swr[D][LD], sredf[NW];
    __shared__ int sbad;
    // ---- stage: the statistics row, the S0 of every cluster (pi), shift / scale ----
    const double* s = stats + (size_t)k * F;
    for (int f = tid; f < F; f += T) sS[f] = s[f];
    double part = 0.0;
    for (int kk = tid; kk < K; kk += T) part += (double)(float)stats[(size_t)kk * F];
    double shift_d = 0.0;
    if (tid < D) { shift_d = (double)shift_f[tid]; sscale[tid] = scale[tid]; }
    const float av = avgvar[k];
    double ll_slot = 0.0;
    if (k == 0 && tid == 0) ll_slot = stats[(size_t)K * F];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((tid & 31) == 0) sredd[tid >> 5] = part;
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
    // ---- pi (compute_pi, gaussian_kernel.cu:172-193), means (gaussian.cu:611-622), R (:663-679, gaussian_kernel.cu:658-675) ----
    double sumN = 0.0;
#pragma unroll
    for (int w = 0; w < NW; w++) sumN += sredd[w];
    const float pik = Nf < 0.5f ? 1e-10f : (float)((double)Nf / sumN);
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
                double cov = (Nf >= 1.0f) ? sS[1 + D + i * (i + 1) / 2 + j] - mi * sS[1 + j] : 0.0;
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
    __syncthreads();
    FIN_STAMP(4);
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
    TC_CUDA_TRY(cudaGetLastError());
    t->e_NG = (K + 15) / 16;
    return GMM_OK;
}

template <int D>
static int launch_estep_d(TcState* t, int K, double* d_ll, cudaStream_t stream) {
    using C = ECfg<D>;
    static_assert(C::SMEM_BYTES <= 232448, "shared memory budget");
    if (!t->attr_estep) {
        TC_CUDA_TRY(cudaFuncSetAttribute(estep_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
        t->attr_estep = true;
    }
    const int ntiles = (t->n + 127) / 128;
    int grid = t->num_sms;
    if (grid > ntiles) grid = ntiles;
    if (grid < 1) grid = 1;
    const int NP = (K + 63) / 64;
    if (NP > 1 && !t->d_den) return fail(GMM_ERR_STATE, "tensor E-step: context was created for at most 64 clusters");
    // P passes of 64 clusters: log-denominators of passes 0 .. P-2 (mode 1), then the last pass writes its final
    // responsibilities and the events' total log-denominators (mode 2, or mode 0 when P = 1), then passes 0 .. P-2 write
    // theirs against those totals (mode 3): 2P - 1 launches, every responsibility stored once
    auto launch = [&](int p, int mode, const float* den_in, float* den_out) {
        const int Kp = K - 64 * p < 64 ? K - 64 * p : 64;
        estep_tc_kernel<D><<<grid, C::THREADS, C::SMEM_BYTES, stream>>>(
            t->d_x, t->d_bimg + (size_t)p * C::MAXSG * C::B_SG, t->d_ck + 128 * p, t->d_shift_f, t->d_inv_scale_f,
            t->d_memb + (size_t)(64 * p) * t->memb_pitch, t->memb_pitch, t->n, Kp, (Kp + C::GB - 1) / C::GB, d_ll, mode, den_in, den_out);
        return cudaGetLastError();
    };
    if (NP == 1) TC_CUDA_TRY(launch(0, 0, nullptr, nullptr));
    else {
        for (int p = 0; p + 1 < NP; p++) TC_CUDA_TRY(launch(p, 1, p ? t->d_den : nullptr, t->d_den));
        TC_CUDA_TRY(launch(NP - 1, 2, t->d_den, t->d_den));
        for (int p = 0; p + 1 < NP; p++) TC_CUDA_TRY(launch(p, 3, t->d_den, nullptr));
    }
    return GMM_OK;
}

int tc_launch_estep(TcState* t, int K, double* d_ll, cudaStream_t stream) {
    if (!t || !t->emap_ok) return fail(GMM_ERR_STATE, "tensor E-step not initialised for this shape");
    switch (t->D) {
        case 8: return launch_estep_d<8>(t, K, d_ll, stream);
        case 16: return launch_estep_d<16>(t, K, d_ll, stream);
        case 24: return launch_estep_d<24>(t, K, d_ll, stream);
        default: return fail(GMM_ERR_ARG, "tensor E-step: unsupported D");
    }
}

template <int D>
static int launch_mstep_d(TcState* t, int K, double* d_stats, cudaStream_t stream) {
    using C = MCfg<D>;
    static_assert(C::SMEM_BYTES <= 232448, "shared memory budget");
    if (!t->attr_mstep) {
        TC_CUDA_TRY(cudaFuncSetAttribute(mstep_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
        t->attr_mstep = true;
    }
    int gx = t->num_sms;
    int per = (t->n + gx - 1) / gx;
    per = (per + kTE - 1) / kTE * kTE;
    gx = (t->n + per - 1) / per;
    const int gy = (K + kNCL - 1) / kNCL;
    if ((size_t)gx * gy * C::MT * 128 * kNCL > t->scratch_floats) return fail(GMM_ERR_STATE, "tensor M-step scratch too small");
    dim3 grid(gx, gy);
    mstep_tc_kernel<D><<<grid, C::THREADS, C::SMEM_BYTES, stream>>>(t->tm_x, t->tm_g, t->n, t->d_scratch, per, t->magic);
    TC_CUDA_TRY(cudaGetLastError());
    mstep_tc_finalize_kernel<<<C::NCHUNK * 8, 256, 0, stream>>>(t->d_scratch, gx, C::MT, K, C::F, t->d_rowmap, t->d_scale, d_stats);
    TC_CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

int tc_launch_mstep(TcState* t, int K, double* d_stats, cudaStream_t stream) {
    if (!t || !t->maps_ok) return fail(GMM_ERR_STATE, "tensor-core M-step not initialised for this shape");
    if (!t->have_shift) return fail(GMM_ERR_STATE, "tensor-core M-step needs gmm_seed (shift/scale) first");
    if (!t->mstep_ready) return fail(GMM_ERR_STATE, "tensor-core M-step: the data range exceeds the fixed-point operand budget");
    switch (t->D) {
        case 4: return launch_mstep_d<4>(t, K, d_stats, stream);
        case 8: return launch_mstep_d<8>(t, K, d_stats, stream);
        case 12: return launch_mstep_d<12>(t, K, d_stats, stream);
        case 16: return launch_mstep_d<16>(t, K, d_stats, stream);
        case 20: return launch_mstep_d<20>(t, K, d_stats, stream);
        case 24: return launch_mstep_d<24>(t, K, d_stats, stream);
        default: return fail(GMM_ERR_ARG, "tensor-core M-step: unsupported D");
    }
}

}  // namespace gmm
