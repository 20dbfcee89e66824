// tc_ptx.cuh — thin inline-PTX wrappers for the Hopper (sm_90a) features the
// tensor-core kernels use: mbarrier, TMA bulk copies (cp.async.bulk), warpgroup
// MMA (wgmma.mma_async / fence / commit / wait), proxy fences.  Descriptor bit
// layouts follow the PTX ISA "matrix descriptor" table of wgmma.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace gmm { namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Arrive whose issue DEPENDS on `dep`: the arrival count operand is selected by a comparison of dep's bit pattern with
// one that no finite or infinite sum produces (a signalling NaN), so it is always 1 — but neither ptxas nor the hardware
// can know that, and the arrive cannot issue before dep (and every load dep was computed from) is in its register.
// Used to hand a shared-memory stage back to a producer only after this warp's loads from it have landed: a plain
// mbarrier.arrive does not wait for the warp's outstanding LDS (measured in round 1, DESIGN.md).
__device__ __forceinline__ void mbar_arrive_after(uint64_t* bar, float dep) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .b32 cnt;\n\t"
        "setp.ne.b32 p, %1, 0xff800001;\n\t"
        "selp.b32 cnt, 1, 2, p;\n\t"
        "mbarrier.arrive.shared::cta.b64 _, [%0], cnt;\n\t}"
        ::"r"(smem_u32(bar)), "r"(__float_as_uint(dep)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// Same, but lets the hardware park the thread for up to `ns` nanoseconds per probe: a waiting
// warp then issues far fewer TRYWAIT/BRA pairs and leaves the issue slots to the warps that work.
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(ns) : "memory");
    }
}
// ---- proxy fences -----------------------------------------------------------
// Generic-proxy shared-memory writes -> visible to the async proxy (TMA, wgmma operands).
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA: 1-D bulk copy global -> shared, completion on an mbarrier -----------
// bytes must be a multiple of 16; src and dst 16-byte aligned.  (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- descriptors ------------------------------------------------------------
// Shared-memory matrix descriptor of wgmma, no swizzle ("interleaved" core-matrix layout):
//   bits [0,14)  start address >> 4
//   bits [16,30) leading-dimension byte offset >> 4  (distance between core matrices adjacent in K)
//   bits [32,46) stride-dimension byte offset >> 4   (distance between core matrices adjacent in M/N)
//   bits [49,52) base offset = 0;  bits [62,64) layout type = 0 (no swizzle)
// A core matrix is 8 rows x 16 bytes, stored as 128 contiguous bytes.
//   K-major  operand: element (r, k)  at (r/8)*SBO + (k_bytes/16)*LBO + (r%8)*16 + k_bytes%16
//   MN-major operand: element (mn, k) at (mn_bytes/16)*SBO + (k/8)*LBO + (k%8)*16 + mn_bytes%16
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// ---- warpgroup MMA ------------------------------------------------------------
// Accumulator fragment of an m64nN f32 result, thread t of the warpgroup (warp w = t/32, lane l):
//   d[i] -> row 16w + l/4 + 8*((i/2)%2), column 8*(i/4) + 2*(l%4) + i%2
// A fragment from registers (f16, m64k16): a0 = row l/4 cols {2q, 2q+1}, a1 = row l/4+8 same cols,
//   a2 / a3 = the same rows at cols {8+2q, 9+2q}   (rows offset by 16w, q = l%4)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 128] (+)= A[64 x 16] (registers, K-major fragments) * B[16 x 128] (shared memory, K-major); one warpgroup.
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc, bool accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc), "r"((uint32_t)accumulate));
}

// D[64 x 64] += A[64 x 16] * B[16 x 64], both from shared memory: A MN-major (transposed), B K-major; one warpgroup.
__device__ __forceinline__ void wgmma_m64n64k16_ss_tn(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc));
}

// D[64 x 32] += A[64 x 16] * B[16 x 32], both from shared memory: A MN-major (transposed), B K-major; one warpgroup.
__device__ __forceinline__ void wgmma_m64n32k16_ss_tn(float (&d)[16], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// pack two floats into half2 bits (round to nearest even): low half = a, high half = b
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}

// 2^x, MUFU.EX2 (denormal results flush to zero; callers pass x <= 0)
__device__ __forceinline__ float ex2_approx(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

}}  // namespace gmm::ptx
