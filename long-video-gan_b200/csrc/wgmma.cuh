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

// D[64 x N] += A[64 x 16] * B[16 x N], N = 16, 32, ..., 256, fp16 or bf16 operands from shared memory, fp32 accumulators in
// registers, issued by the whole warpgroup. TA / TB: 0 = K-major, 1 = MN-major. Fragment of thread t (warp w = t / 32 of the
// warpgroup, lane l): d[4 j + r] = D[16 w + l / 4 + 8 (r / 2)][8 j + 2 (l % 4) + r % 2], j < N / 8 -- the concatenation of
// the fragments of N / 8 consecutive 8-column slices, whatever N is.
#define LVG_D8(i)                                                                                                            \
    "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// NS: N as a string; REGS: the accumulator list; A0 .. SC: operand numbers of a_lo, a_hi, b_lo, b_hi, TA, TB, scale-d
#define LVG_WGMMA_ASM(NS, TYPE, REGS, A0, A1, B0, B1, TA_, TB_, SC)                                                           \
    "{\n .reg .b64 da, db;\n .reg .pred p;\n setp.ne.b32 p, %" SC ", 0;\n mov.b64 da, {%" A0 ", %" A1 "};\n"                   \
    " mov.b64 db, {%" B0 ", %" B1 "};\n wgmma.mma_async.sync.aligned.m64n" NS "k16.f32." TYPE "." TYPE " " REGS                 \
    ", da, db, p, 1, 1, %" TA_ ", %" TB_ ";\n}\n"
#define LVG_WGMMA(NS, REGS, A0, A1, B0, B1, TA_, TB_, SC, ...)                                                                \
    do {                                                                                                                       \
        if constexpr (BF16)                                                                                                    \
            asm volatile(LVG_WGMMA_ASM(NS, "bf16", REGS, A0, A1, B0, B1, TA_, TB_, SC)                                        \
                         : __VA_ARGS__ : "r"(a_lo), "r"(a_hi), "r"(b_lo), "r"(b_hi), "n"(TA), "n"(TB), "r"(1));               \
        else                                                                                                                   \
            asm volatile(LVG_WGMMA_ASM(NS, "f16", REGS, A0, A1, B0, B1, TA_, TB_, SC)                                         \
                         : __VA_ARGS__ : "r"(a_lo), "r"(a_hi), "r"(b_lo), "r"(b_hi), "n"(TA), "n"(TB), "r"(1));               \
    } while (0)
template <bool BF16, int N, int TA, int TB>
__device__ __forceinline__ void wgmma_m64nNk16(float (&d)[N / 2], uint32_t a_lo, uint32_t a_hi, uint32_t b_lo, uint32_t b_hi)
{
    static_assert(N % 16 == 0 && N >= 16 && N <= 256, "wgmma: N = 16, 32, ..., 256");
    // ---- BEGIN GENERATED (tools/gen_wgmma.py)
    if constexpr (N == 16) LVG_WGMMA("16", "{%0, %1, %2, %3, %4, %5, %6, %7}", "8", "9", "10", "11", "12", "13", "14", LVG_D8(0));
    else if constexpr (N == 32) LVG_WGMMA("32", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}", "16", "17", "18", "19", "20", "21", "22", LVG_D8(0), LVG_D8(8));
    else if constexpr (N == 48) LVG_WGMMA("48", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}", "24", "25", "26", "27", "28", "29", "30", LVG_D8(0), LVG_D8(8), LVG_D8(16));
    else if constexpr (N == 64) LVG_WGMMA("64", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}", "32", "33", "34", "35", "36", "37", "38", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24));
    else if constexpr (N == 80) LVG_WGMMA("80", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}", "40", "41", "42", "43", "44", "45", "46", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32));
    else if constexpr (N == 96) LVG_WGMMA("96", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}", "48", "49", "50", "51", "52", "53", "54", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40));
    else if constexpr (N == 112) LVG_WGMMA("112", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}", "56", "57", "58", "59", "60", "61", "62", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48));
    else if constexpr (N == 128) LVG_WGMMA("128", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}", "64", "65", "66", "67", "68", "69", "70", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56));
    else if constexpr (N == 144) LVG_WGMMA("144", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}", "72", "73", "74", "75", "76", "77", "78", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64));
    else if constexpr (N == 160) LVG_WGMMA("160", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}", "80", "81", "82", "83", "84", "85", "86", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72));
    else if constexpr (N == 176) LVG_WGMMA("176", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87}", "88", "89", "90", "91", "92", "93", "94", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72), LVG_D8(80));
    else if constexpr (N == 192) LVG_WGMMA("192", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}", "96", "97", "98", "99", "100", "101", "102", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72), LVG_D8(80), LVG_D8(88));
    else if constexpr (N == 208) LVG_WGMMA("208", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103}", "104", "105", "106", "107", "108", "109", "110", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72), LVG_D8(80), LVG_D8(88), LVG_D8(96));
    else if constexpr (N == 224) LVG_WGMMA("224", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111}", "112", "113", "114", "115", "116", "117", "118", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72), LVG_D8(80), LVG_D8(88), LVG_D8(96), LVG_D8(104));
    else if constexpr (N == 240) LVG_WGMMA("240", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119}", "120", "121", "122", "123", "124", "125", "126", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72), LVG_D8(80), LVG_D8(88), LVG_D8(96), LVG_D8(104), LVG_D8(112));
    else if constexpr (N == 256) LVG_WGMMA("256", "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}", "128", "129", "130", "131", "132", "133", "134", LVG_D8(0), LVG_D8(8), LVG_D8(16), LVG_D8(24), LVG_D8(32), LVG_D8(40), LVG_D8(48), LVG_D8(56), LVG_D8(64), LVG_D8(72), LVG_D8(80), LVG_D8(88), LVG_D8(96), LVG_D8(104), LVG_D8(112), LVG_D8(120));
    // ---- END GENERATED
}
#undef LVG_WGMMA
#undef LVG_WGMMA_ASM
#undef LVG_D8

}  // namespace tc
}  // namespace lvg
