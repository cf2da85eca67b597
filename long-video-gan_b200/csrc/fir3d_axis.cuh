// One axis of the separable 4-tap FIR of fir3d.cu and dblock_tail.cu, and the tile both kernels walk.
//
// Per axis the operator P is a copy or   out[m] = sum_j g[j] * in[step * m + off + j]   (g[j] = f[3 - j], samples outside
// [0, n_in) are zero), step 1 or 2. The adjoint gathers   out[m] = sum over (i, j) with step * i + off + j == m of
// g[j] * in[i].
#pragma once

#include "common.cuh"

namespace lvg {
namespace fir3d_axis {

constexpr int kTH = 8, kTW = 32, kThreads = kTH * kTW;
constexpr int kRows = 2 * (kTH - 1) + 4;      // input rows one tile reads (step 2, 4 taps)
constexpr int kCols = 2 * (kTW - 1) + 4;
constexpr int kLoads = (kRows * kCols + kThreads - 1) / kThreads;

struct Axis {
    int filt, step, off, n_in, n_out;         // as the operator P sees them; the adjoint runs n_out -> n_in
};

// first input index and taps of output m along one axis; the taps are in[base + r], r < ntaps(a)
template <bool ADJ> __device__ __forceinline__ int ax_base(const Axis& a, int m) {
    if (!a.filt) return m;
    if (!ADJ) return a.step * m + a.off;
    return a.step == 1 ? m - a.off - 3 : ((m - a.off) >> 1) - 1;
}
template <bool ADJ> __device__ __forceinline__ int ax_ntaps(const Axis& a) {
    return !a.filt ? 1 : (ADJ && a.step == 2) ? 2 : 4;
}
template <bool ADJ> __device__ __forceinline__ float ax_tap(const Axis& a, const float (&g)[4], int m, int r) {
    if (!a.filt) return 1.f;
    if (!ADJ) return g[r];
    if (a.step == 1) return g[3 - r];
    const bool odd = (m - a.off) & 1;         // in[q - 1] carries tap jp + 2, in[q] tap jp (jp = odd)
    return r == 0 ? (odd ? g[3] : g[2]) : (odd ? g[1] : g[0]);
}

}  // namespace fir3d_axis
}  // namespace lvg
