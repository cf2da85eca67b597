// The conditioning of a super-res generator layer by its per-axis plan (DESIGN.md 7h), shared by the two kernels that
// evaluate it: sres_cond_kernel (csrc/sres_cond.cu, writes the layer input z) and conv_pack_cond_kernel (csrc/conv_igemm.cu,
// writes the convolution's re-tiled operand straight from x_prev and the low-res video). Both take the tap tables, the
// vertical pass and the horizontal pass from here, so their sums run in the same order and round to the same bits.
//
// Along an axis, output index i reads the resampler output m = x0 + clamp(i - px0, 0, mhi); that is
// gain * sum_k f[K - 1 - k] * zu[m down + k - pad0] over the zero-upsampled (by `up`) replicate-padded frame, zero outside
// [0, zlen), and sample v = j / up of that frame is low-res row / column clamp(v - shift, 0, len - 1). Identity axes: K = 0.
#pragma once

#include "common.cuh"

namespace lvg {
namespace sres {

constexpr int kMaxTaps = 64;                 // filter taps per axis

struct Axis {
    int out, px0, mhi, x0, up, down, pad0, zlen, shift, ntaps, len;
    int nt;                                  // taps per output: ceil(ntaps / up), 1 for identity
    float gain;
    const float* f;
};

// taps of output index i along an axis: (source index, weight) for each of a.nt slots, weight 0 where unused
__device__ __forceinline__ void axis_taps(const Axis& a, int i, int* src, float* wgt)
{
    const int m = a.x0 + min(max(i - a.px0, 0), a.mhi);
    if (a.ntaps == 0) {
        src[0] = min(max(m - a.shift, 0), a.len - 1);
        wgt[0] = 1.f;
        return;
    }
    const int base = m * a.down - a.pad0;                    // zu index of tap k = base + k
    int k = ((-base) % a.up + a.up) % a.up;                   // first tap on a nonzero (non-inserted) sample
    int slot = 0;
    for (; k < a.ntaps; k += a.up, slot++) {
        const int j = base + k;
        const bool in = j >= 0 && j < a.zlen;
        const int v = in ? j / a.up : 0;
        src[slot] = min(max(v - a.shift, 0), a.len - 1);
        wgt[slot] = in ? a.gain * __ldg(a.f + a.ntaps - 1 - k) : 0.f;
    }
    for (; slot < a.nt; slot++) {
        src[slot] = 0;
        wgt[slot] = 0.f;
    }
}

// vertical pass at low-res column x of one output row: sum_k wh[k] L[sh[k]][x] (nth taps, zero weights skipped)
__device__ __forceinline__ float vertical_tap_sum(const float* __restrict__ L, int64_t s_h, int64_t s_w, int x, const float* wh,
                                                  const int* sh, int nth)
{
    float acc = 0.f;
    for (int k = 0; k < nth; k++) {
        const float wk = wh[k];
        if (wk != 0.f) acc += wk * __ldg(L + sh[k] * s_h + x * s_w);
    }
    return acc;
}

// horizontal pass of one output pixel over the vertical pass's row: sum_k ww[k] row[sw[k]] (ntw taps, zero weights skipped)
__device__ __forceinline__ float horizontal_tap_sum(const float* row, const float* ww, const int* sw, int ntw)
{
    float acc = 0.f;
    for (int k = 0; k < ntw; k++) {
        const float wk = ww[k];
        if (wk != 0.f) acc += wk * row[sw[k]];
    }
    return acc;
}

// one axis of a plan (LVG_SRES_COND_NPLAN ints) checked against what the kernels index; false outside the envelope
inline bool read_axis(const int* q, int len, Axis& a)
{
    a.out = q[0]; a.px0 = q[1]; a.mhi = q[2]; a.x0 = q[3]; a.up = q[4]; a.down = q[5]; a.pad0 = q[6]; a.zlen = q[7];
    a.shift = q[8]; a.ntaps = q[9]; a.len = len;
    if (a.out < 1 || a.out > (1 << 20) || a.mhi < 0 || a.x0 < 0 || a.up < 1 || a.down < 1 || a.zlen < 1 || len < 1
        || a.ntaps < 0 || a.ntaps > kMaxTaps || a.up > kMaxTaps || a.down > kMaxTaps)
        return false;
    if (a.ntaps == 0 && (a.up != 1 || a.down != 1 || a.pad0 != 0)) return false;
    a.nt = a.ntaps == 0 ? 1 : (a.ntaps + a.up - 1) / a.up;
    // every index the kernels form stays far inside int
    const int64_t mmax = (int64_t)a.x0 + a.mhi;
    if (mmax * a.down + a.ntaps + (a.pad0 < 0 ? -(int64_t)a.pad0 : (int64_t)a.pad0) > (1 << 28)) return false;
    if (a.px0 < -(1 << 20) || a.px0 > (1 << 20) || a.shift < -(1 << 20) || a.shift > (1 << 20)) return false;
    return true;
}

}  // namespace sres
}  // namespace lvg
