// Shared helpers for the liblvg_ops kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/lvg_ops.h"

#ifndef __CUDA_ARCH_LIST__
#endif

namespace lvg {

// ---------------------------------------------------------------------------
// Error reporting (thread local, read through lvg_last_error()).

void set_error(const char* fmt, ...);

#define LVG_REQUIRE(cond, ...)                              \
    do {                                                    \
        if (!(cond)) {                                      \
            ::lvg::set_error(__VA_ARGS__);                  \
            return LVG_ERR_ARG;                             \
        }                                                   \
    } while (0)

#define LVG_CUDA(expr)                                                        \
    do {                                                                      \
        cudaError_t e__ = (expr);                                             \
        if (e__ != cudaSuccess) {                                             \
            ::lvg::set_error("%s failed: %s (%s:%d)", #expr,                  \
                             cudaGetErrorString(e__), __FILE__, __LINE__);    \
            return LVG_ERR_CUDA;                                              \
        }                                                                     \
    } while (0)

// after every kernel launch: count it (lvg_launch_count) and pick up configuration errors without synchronising
void count_launch();
#define LVG_LAUNCH_CHECK()                  \
    do {                                    \
        ::lvg::count_launch();              \
        LVG_CUDA(cudaPeekAtLastError());    \
    } while (0)

inline int num_sms() {
    static int cached[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (cached[dev] == 0) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        cached[dev] = v > 0 ? v : 132;
    }
    return cached[dev];
}

inline size_t dtype_size(int dtype) {
    return dtype == LVG_F16 ? 2 : dtype == LVG_F64 ? 8 : 4;
}

// ---------------------------------------------------------------------------
// Arithmetic type used inside kernels: fp16 and fp32 storage compute in fp32,
// fp64 in fp64 (the reference's InternalType, bias_act.cu:15-18).

template <class T> struct Acc { typedef float type; };
template <> struct Acc<double> { typedef double type; };

template <class T> __device__ __forceinline__ typename Acc<T>::type to_acc(T v) { return (typename Acc<T>::type)v; }
template <> __device__ __forceinline__ float to_acc<__half>(__half v) { return __half2float(v); }

template <class T> __device__ __forceinline__ T from_acc(typename Acc<T>::type v) { return (T)v; }
template <> __device__ __forceinline__ __half from_acc<__half>(float v) { return __float2half_rn(v); }

// ---------------------------------------------------------------------------
// 128-bit vector access. VecOf<T>::N elements of T in one 16-byte word.

template <class T> struct VecOf;
template <> struct VecOf<float>  { static constexpr int N = 4; };
template <> struct VecOf<__half> { static constexpr int N = 8; };
template <> struct VecOf<double> { static constexpr int N = 2; };

template <class T> struct alignas(16) Pack { T v[VecOf<T>::N]; };

template <class T> __device__ __forceinline__ Pack<T> load_pack(const T* p) {
    Pack<T> r;
    *reinterpret_cast<uint4*>(&r) = __ldg(reinterpret_cast<const uint4*>(p));
    return r;
}
template <class T> __device__ __forceinline__ void store_pack(T* p, const Pack<T>& v) {
    *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&v);
}

// whole-pack conversions; fp16 goes through the paired cvt instructions (half2 <-> float2)
template <class T> __device__ __forceinline__ void unpack(const Pack<T>& p, typename Acc<T>::type (&f)[VecOf<T>::N]) {
#pragma unroll
    for (int k = 0; k < VecOf<T>::N; k++) f[k] = to_acc(p.v[k]);
}
template <> __device__ __forceinline__ void unpack<__half>(const Pack<__half>& p, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&p);
#pragma unroll
    for (int k = 0; k < 4; k++) { const float2 t = __half22float2(h[k]); f[2 * k] = t.x; f[2 * k + 1] = t.y; }
}
template <class T> __device__ __forceinline__ Pack<T> pack(const typename Acc<T>::type (&f)[VecOf<T>::N]) {
    Pack<T> p;
#pragma unroll
    for (int k = 0; k < VecOf<T>::N; k++) p.v[k] = from_acc<T>(f[k]);
    return p;
}
template <> __device__ __forceinline__ Pack<__half> pack<__half>(const float (&f)[8]) {
    Pack<__half> p;
    __half2* h = reinterpret_cast<__half2*>(&p);
#pragma unroll
    for (int k = 0; k < 4; k++) h[k] = __floats2half2_rn(f[2 * k], f[2 * k + 1]);
    return p;
}

__host__ __device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// floor division / positive modulo for possibly negative numerators
__host__ __device__ __forceinline__ int floordiv(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
__host__ __device__ __forceinline__ int posmod(int a, int b) { int r = a % b; return r < 0 ? r + b : r; }
__host__ __device__ __forceinline__ int ceildiv(int a, int b) { return floordiv(a + b - 1, b); }

}  // namespace lvg
