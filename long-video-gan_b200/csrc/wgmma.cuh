// wgmma / mbarrier / bulk-copy PTX wrappers shared by the tensor-core convolution kernels (sm_90a).
#pragma once
#include "common.cuh"

namespace lvg {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// one lane of a converged warp (elect.sync): the compiler knows a single thread is active behind this predicate and
// issues the TMA instructions straight, without wrapping each in an election loop
__device__ __forceinline__ bool elect_one()
{
    uint32_t pred = 0;
    asm volatile(
        "{\n"
        " .reg .pred p;\n"
        " elect.sync _|p, 0xffffffff;\n"
        " selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// the spin loop lives inside the asm, so no C++ loop surrounds the MMAs that follow a wait
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        " .reg .pred p;\n"
        "LVG_WAIT_%=:\n"
        " mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        " @!p bra LVG_WAIT_%=;\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// mbar_arrive by the threads with `pred` set, as a predicated instruction (no branch around it)
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred)
{
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %1, 0;\n @p mbarrier.arrive.shared::cta.b64 _, [%0];\n}\n" ::"r"(smem_u32(bar)), "r"((int)pred)
                 : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// 1-D bulk copy global -> shared through the TMA engine; completion is signalled on `bar` (complete_tx)
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Shared-memory matrix descriptor of wgmma, no swizzle ("interleave" canonical layouts of 8-row x 16-byte core matrices):
// start address, leading / stride byte offsets, all >> 4. K-major operands: LBO = step between the two 8-element K halves,
// SBO = step between 8-row groups along M / N. MN-major operands: LBO = step between 8-row groups along K, SBO = step
// between 8-element groups along M / N.
// As two 32-bit words, so that the issuing loops step through K / taps with ONE 32-bit add on the low word (start
// address >> 4 in bits 0-13; shared-memory addresses stay below 256 KB, so the sum never carries into the LBO field).
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo_bytes) { return ((saddr >> 4) & 0x3fffu) | (((lbo_bytes >> 4) & 0x3fffu) << 16); }
__device__ __forceinline__ uint32_t desc_hi(uint32_t sbo_bytes) { return (sbo_bytes >> 4) & 0x3fffu; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 64] += A[64 x 16] * B[16 x 64], fp16 or bf16 operands from shared memory, fp32 accumulators in registers, issued by
// the whole warpgroup. TA / TB: 0 = K-major, 1 = MN-major. Fragment of thread t (warp w = t / 32 of the warpgroup, lane l):
// d[4 j + r] = D[16 w + l / 4 + 8 (r / 2)][8 j + 2 (l % 4) + r % 2].
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint32_t a_lo, uint32_t a_hi, uint32_t b_lo, uint32_t b_hi)
{
#define LVG_WGMMA_N64(TYPE)                                                                                                        \
    asm volatile(                                                                                                                  \
        "{\n"                                                                                                                      \
        " .reg .b64 da, db;\n"                                                                                                     \
        " .reg .pred p;\n"                                                                                                         \
        " setp.ne.b32 p, %38, 0;\n"                                                                                                \
        " mov.b64 da, {%32, %33};\n"                                                                                               \
        " mov.b64 db, {%34, %35};\n"                                                                                               \
        " wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPE "." TYPE " "                                                           \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                                  \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, da, db, p, 1, 1, %36, %37;\n"            \
        "}\n"                                                                                                                      \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),    \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),    \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])                                                                       \
        : "r"(a_lo), "r"(a_hi), "r"(b_lo), "r"(b_hi), "n"(TA), "n"(TB), "r"(1))
    if constexpr (BF16) LVG_WGMMA_N64("bf16");
    else LVG_WGMMA_N64("f16");
#undef LVG_WGMMA_N64
}

// the same with N = 32 (d[4 j + r] as above, j < 4)
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint32_t a_lo, uint32_t a_hi, uint32_t b_lo, uint32_t b_hi)
{
#define LVG_WGMMA_N32(TYPE)                                                                                                        \
    asm volatile(                                                                                                                  \
        "{\n"                                                                                                                      \
        " .reg .b64 da, db;\n"                                                                                                     \
        " .reg .pred p;\n"                                                                                                         \
        " setp.ne.b32 p, %22, 0;\n"                                                                                                \
        " mov.b64 da, {%16, %17};\n"                                                                                               \
        " mov.b64 db, {%18, %19};\n"                                                                                               \
        " wgmma.mma_async.sync.aligned.m64n32k16.f32." TYPE "." TYPE " "                                                           \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, da, db, p, 1, 1, %20, %21;\n"                     \
        "}\n"                                                                                                                      \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])                                             \
        : "r"(a_lo), "r"(a_hi), "r"(b_lo), "r"(b_hi), "n"(TA), "n"(TB), "r"(1))
    if constexpr (BF16) LVG_WGMMA_N32("bf16");
    else LVG_WGMMA_N32("f16");
#undef LVG_WGMMA_N32
}

}  // namespace tc
}  // namespace lvg
