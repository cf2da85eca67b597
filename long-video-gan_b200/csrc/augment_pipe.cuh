// The coordinate and weight function of ADA's geometric augmentation (AugmentPipe, DESIGN.md 7e), shared by the forward and
// adjoint kernels of augment_pipe.cu and by the host emulation tools/augment_pipe_emul.cu. Every rounding step is explicit
// (no contraction left to the compiler), so host and device builds compute the same fp32 values.
//
// Per axis, v point j of a v extent nv samples u (the 2x upsampled, reflect-padded x, extent lu = 2 * padded size) at
//   c = ((g + 1) * lu - 1) / 2,   g = theta . (base(j), base(i), 1),   base = affine_grid's align_corners=False grid;
// the bilinear sample of u at c is a 7-tap window of xpad from i0 = floor(floor(c) / 2) - 3 (axis_of / tap).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define AP_HD __host__ __device__ __forceinline__
#else
#define AP_HD inline
#endif

namespace lvg {
namespace ap {

constexpr int kTaps = 12;       // Hz_geom: sym6, 12 taps
constexpr int kWin = 7;         // xpad taps of one bilinear sample of u, per axis
constexpr int kNpar = 23;       // mx0, my0, mx1, my1, theta[6], C[3][4], sigma

AP_HD float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
AP_HD float add_rn(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
AP_HD float fma_rn(float a, float b, float c) {
#ifdef __CUDA_ARCH__
    return __fmaf_rn(a, b, c);
#else
    return fmaf(a, b, c);
#endif
}
AP_HD int floor_div2(int a) { return a >= 0 ? a / 2 : -((1 - a) / 2); }

// affine_grid's base coordinate of point i of n (align_corners=False): linspace(-1, 1, n) * (n - 1) * fp32(1 / n), the
// CUDA arithmetic (linspace fills from both ends; a division by a scalar is a multiplication by its reciprocal)
AP_HD float grid_base(int i, int n) {
    const float step = 2.f / (float)(n - 1);
    const float lin = i < n / 2 ? fma_rn(step, (float)i, -1.f) : fma_rn(-step, (float)(n - 1 - i), 1.f);
    return mul_rn(mul_rn(lin, (float)(n - 1)), 1.f / (float)n);
}

// sampling coordinates in u of the v point with base coordinates (xb, yb); th = theta row-major [2][3]
AP_HD void point_coord(const float* th, float xb, float yb, int lux, int luy, float& ix, float& iy) {
    const float gx = add_rn(fma_rn(yb, th[1], mul_rn(xb, th[0])), th[2]);
    const float gy = add_rn(fma_rn(yb, th[4], mul_rn(xb, th[3])), th[5]);
    ix = mul_rn(fma_rn(add_rn(gx, 1.f), (float)lux, -1.f), 0.5f);
    iy = mul_rn(fma_rn(add_rn(gy, 1.f), (float)luy, -1.f), 0.5f);
}

// one axis of a bilinear sample of u at c: window base i0 in xpad, parity r of floor(c), and the weights of the two u taps
// floor(c) and floor(c) + 1 (zero for a tap outside [0, lu): grid_sample's zero padding)
struct Axis {
    int i0, r;
    float a0, a1;
};

AP_HD Axis axis_of(float c, int lu) {
    Axis ax{0, 0, 0.f, 0.f};
    const float fl = floorf(c);
    if (!(fl >= -1.f && fl < (float)lu)) return ax;          // both taps outside u (or c is NaN)
    const int x0 = (int)fl;
    if (x0 >= 0) ax.a0 = add_rn(add_rn(fl, 1.f), -c);
    if (x0 + 1 < lu) ax.a1 = add_rn(c, -fl);
    ax.i0 = floor_div2(x0) - 3;
    ax.r = x0 - 2 * floor_div2(x0);
    return ax;
}

// weight of xpad[i0 + k] (0 <= k < 7) in the sample: 2 ((1 - a) f[11 + r - 2k] + a f[12 + r - 2k]), f zero outside 0..11
AP_HD float tap(const Axis& ax, int k, const float* f) {
    const int j0 = 11 + ax.r - 2 * k;
    float w = 0.f;
    if (j0 >= 0 && j0 < kTaps) w = mul_rn(ax.a0, f[j0]);
    if (j0 + 1 >= 0 && j0 + 1 < kTaps) w = fma_rn(ax.a1, f[j0 + 1], w);
    return mul_rn(w, 2.f);
}

// x index of xpad index i (0 <= i < len + m0 + m1, margins <= len - 1: one reflection), clamped for safety
AP_HD int reflect(int i, int m0, int len) {
    int j = i - m0;
    j = j < 0 ? -j : (j >= len ? 2 * (len - 1) - j : j);
    return j < 0 ? 0 : (j >= len ? len - 1 : j);
}

// the xpad indices that hold x index j: a = 0 itself, a = 1 its reflection on the low side, a = 2 on the high side;
// -1 where that reflection is not in the padded frame
AP_HD int copy_at(int j, int m0, int m1, int len, int a) {
    if (a == 0) return j + m0;
    if (a == 1) return j >= 1 && j <= m0 ? m0 - j : -1;
    return j <= len - 2 && j > len - 2 - m1 ? m0 + 2 * (len - 1) - j : -1;
}

// The v points whose 7 x 7 window holds xpad point (py, px): floor(c) / 2 - 3 in [p - 6, p], so c in [2p - 6, 2p + 8) on
// both axes. That u-rectangle, widened by half a u pixel against rounding, is mapped back through theta: box_rows gives
// the v rows (plus one row of slack on either side), box_cols the columns of one row (plus one column).
struct Box {
    double gx_lo, gx_hi, gy_lo, gy_hi;
    int vi_lo, vi_hi;
};

AP_HD double g_of(double c, int lu) { return (2.0 * c + 1.0) / lu - 1.0; }

AP_HD int clamp_index(double v, int n) { return v < 0.0 ? 0 : (v > n - 1 ? n - 1 : (int)v); }

AP_HD Box box_rows(const float* th, int px, int py, int lux, int luy, int hv) {
    Box b;
    b.gx_lo = g_of(2.0 * px - 6.5, lux);
    b.gx_hi = g_of(2.0 * px + 8.5, lux);
    b.gy_lo = g_of(2.0 * py - 6.5, luy);
    b.gy_hi = g_of(2.0 * py + 8.5, luy);
    const double det = (double)th[0] * th[4] - (double)th[1] * th[3];
    b.vi_lo = 0;
    b.vi_hi = hv - 1;
    if (fabs(det) < 1e-20) return b;
    double lo = 1e300, hi = -1e300;
    for (int q = 0; q < 4; q++) {
        const double gx = (q & 1 ? b.gx_hi : b.gx_lo) - th[2], gy = (q & 2 ? b.gy_hi : b.gy_lo) - th[5];
        const double yb = (th[0] * gy - th[3] * gx) / det;
        lo = fmin(lo, yb);
        hi = fmax(hi, yb);
    }
    b.vi_lo = clamp_index(floor(((lo + 1.0) * hv - 1.0) / 2.0) - 1.0, hv);
    b.vi_hi = clamp_index(ceil(((hi + 1.0) * hv - 1.0) / 2.0) + 1.0, hv);
    return b;
}

// columns [j_lo, j_hi] of row base yb; false when the row has none
AP_HD bool box_cols(const float* th, const Box& b, float yb, int wv, int& j_lo, int& j_hi) {
    double lo = -1e300, hi = 1e300;
    for (int a = 0; a < 2; a++) {
        const double t0 = th[3 * a], rest = (double)th[3 * a + 1] * yb + th[3 * a + 2];
        const double glo = a ? b.gy_lo : b.gx_lo, ghi = a ? b.gy_hi : b.gx_hi;
        if (t0 == 0.0) {
            if (rest < glo || rest > ghi) return false;
            continue;
        }
        double e0 = (glo - rest) / t0, e1 = (ghi - rest) / t0;
        lo = fmax(lo, fmin(e0, e1));
        hi = fmin(hi, fmax(e0, e1));
    }
    if (lo > hi) return false;
    const double jl = floor(((lo + 1.0) * wv - 1.0) / 2.0) - 1.0, jh = ceil(((hi + 1.0) * wv - 1.0) / 2.0) + 1.0;
    if (jh < 0.0 || jl > wv - 1) return false;
    j_lo = clamp_index(jl, wv);
    j_hi = clamp_index(jh, wv);
    return true;
}

}  // namespace ap
}  // namespace lvg
