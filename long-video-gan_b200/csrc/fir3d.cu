// Separable 4-tap FIR over the T, H and W axes of an NCTHW tensor, and its exact adjoint.
//
// Per axis the operator P is a copy or   out[m] = sum_j g[j] * in[step * m + off + j]   (g[j] = f[3 - j]: convolution
// order, as upfirdn2d with flip_filter = False; samples outside [0, n_in) are zero), step 1 or 2. This is Downsample3d's
// filter (discriminator_lres.py:186-213) at full rate or with step 2, so conv3d_down.py can filter the Cin-channel input of a
// downsampling Conv3dLayer before the convolution instead of its full-resolution output after it. `fold` stores the T axis
// of the filtered side as two phase blocks of channels, t = 2 t' + p -> channel p * C + c, which turns a T-stride-2
// convolution into a T-stride-1 one over 2 C channels.
//
// One CTA owns one (n, c) plane and an 8 x 32 tile of output rows x columns and walks all frames once: each input frame is
// read once, filtered along H then W through shared memory, and the T filter runs over a 4-frame register window. The
// adjoint is the same walk with every axis's gather transposed (out[m] = sum over (i, j) with step * i + off + j == m of
// g[j] * in[i]). fp32 accumulation for fp16 and fp32 storage.
#include "common.cuh"
#include "fir3d_axis.cuh"

namespace lvg {
namespace {

using namespace fir3d_axis;

template <class T, bool ADJ>
__device__ __forceinline__ void fir3d_body(const T* __restrict__ x, const float* __restrict__ f, T* __restrict__ y, int c, int fold,
                                           Axis at, Axis ah, Axis aw)
{
    __shared__ float sa[kRows][kCols + 1];
    __shared__ float sb[kTH][kCols + 1];
    float g[4];
#pragma unroll
    for (int j = 0; j < 4; j++) g[j] = f[3 - j];

    // extents as this kernel reads / writes them
    const int tin = ADJ ? at.n_out : at.n_in, tout = ADJ ? at.n_in : at.n_out;
    const int hin = ADJ ? ah.n_out : ah.n_in, hout = ADJ ? ah.n_in : ah.n_out;
    const int win_ = ADJ ? aw.n_out : aw.n_in, wout = ADJ ? aw.n_in : aw.n_out;

    const int nc = blockIdx.x, n = nc / c, ci = nc - n * c;
    const int tiles_w = (wout + kTW - 1) / kTW;
    const int h0 = (blockIdx.y / tiles_w) * kTH, w0 = (blockIdx.y % tiles_w) * kTW;
    const int h1 = min(h0 + kTH, hout), w1 = min(w0 + kTW, wout);
    const int r_lo = ax_base<ADJ>(ah, h0), c_lo = ax_base<ADJ>(aw, w0);
    const int nrows = ax_base<ADJ>(ah, h1 - 1) + ax_ntaps<ADJ>(ah) - r_lo;
    const int ncols = ax_base<ADJ>(aw, w1 - 1) + ax_ntaps<ADJ>(aw) - c_lo;
    const int nth = ax_ntaps<ADJ>(ah), ntw = ax_ntaps<ADJ>(aw), ntt = ax_ntaps<ADJ>(at);

    const int tid = threadIdx.x, my_r = tid / kTW, my_q = tid % kTW;
    const bool mine = h0 + my_r < h1 && w0 + my_q < w1;
    const int mw = w0 + my_q;
    const int bw = ax_base<ADJ>(aw, mw) - c_lo;
    float tw[4];
#pragma unroll
    for (int r = 0; r < 4; r++) tw[r] = r < ntw ? ax_tap<ADJ>(aw, g, mw, r) : 0.f;

    const int64_t plane_in = (int64_t)hin * win_, plane_out = (int64_t)hout * wout;
    const bool fold_in = fold && ADJ, fold_out = fold && !ADJ;
    auto frame_off = [&](int t, int ext, bool folded, int64_t plane) -> int64_t {
        return folded ? (((int64_t)n * 2 * c + (t & 1) * c + ci) * (ext / 2) + (t >> 1)) * plane
                      : ((int64_t)nc * ext + t) * plane;
    };

    float win[4] = {0.f, 0.f, 0.f, 0.f};     // filtered frames base_t .. base_t + 3 at this thread's output pixel
    int loaded = ax_base<ADJ>(at, 0) - 1;
    for (int mt = 0; mt < tout; mt++) {
        const int bt = ax_base<ADJ>(at, mt);
        while (loaded < bt + 3) {             // block-uniform
            ++loaded;
            float v = 0.f;
            if (loaded >= 0 && loaded < tin) {
                const T* xf = x + frame_off(loaded, tin, fold_in, plane_in);
                float ld[kLoads];
#pragma unroll
                for (int k = 0; k < kLoads; k++) {
                    const int idx = tid + k * kThreads;
                    const int rr = idx / ncols, cc = idx - rr * ncols, gr = r_lo + rr, gc = c_lo + cc;
                    ld[k] = (rr < nrows && gr >= 0 && gr < hin && gc >= 0 && gc < win_) ? to_acc(xf[(int64_t)gr * win_ + gc]) : 0.f;
                }
#pragma unroll
                for (int k = 0; k < kLoads; k++) {
                    const int idx = tid + k * kThreads;
                    const int rr = idx / ncols;
                    if (rr < nrows) sa[rr][idx - rr * ncols] = ld[k];
                }
                __syncthreads();
                for (int idx = tid; idx < kTH * ncols; idx += kThreads) {
                    const int rr = idx / ncols, cc = idx - rr * ncols, m = h0 + rr;
                    float s = 0.f;
                    if (m < h1) {
                        const int b = ax_base<ADJ>(ah, m) - r_lo;
#pragma unroll
                        for (int r = 0; r < 4; r++)
                            if (r < nth) s = fmaf(ax_tap<ADJ>(ah, g, m, r), sa[b + r][cc], s);
                    }
                    sb[rr][cc] = s;
                }
                __syncthreads();
                if (mine) {
#pragma unroll
                    for (int r = 0; r < 4; r++)
                        if (r < ntw) v = fmaf(tw[r], sb[my_r][bw + r], v);
                }
            }
#pragma unroll
            for (int r = 0; r < 3; r++) win[r] = win[r + 1];
            win[3] = v;
        }
        if (mine) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < 4; r++)
                if (r < ntt) s = fmaf(ax_tap<ADJ>(at, g, mt, r), win[r], s);
            y[frame_off(mt, tout, fold_out, plane_out) + (int64_t)(h0 + my_r) * wout + mw] = from_acc<T>(s);
        }
    }
}

template <class T>
__global__ void __launch_bounds__(kThreads) fir3d_down_kernel(const T* __restrict__ x, const float* __restrict__ f, T* __restrict__ y,
                                                             int c, int fold, Axis at, Axis ah, Axis aw)
{
    fir3d_body<T, false>(x, f, y, c, fold, at, ah, aw);
}

template <class T>
__global__ void __launch_bounds__(kThreads) fir3d_adjoint_kernel(const T* __restrict__ x, const float* __restrict__ f, T* __restrict__ y,
                                                                int c, int fold, Axis at, Axis ah, Axis aw)
{
    fir3d_body<T, true>(x, f, y, c, fold, at, ah, aw);
}

int fir3d_launch(bool adj, const void* x, const float* f, void* y, int dtype, int n, int c, const int* in, const int* out,
                 const int* filt, const int* step, const int* off, int fold, void* stream)
{
    const char* name = adj ? "fir3d_adjoint" : "fir3d";
    LVG_REQUIRE(x && f && y, "%s: x, f, y must not be NULL", name);
    LVG_REQUIRE(dtype == LVG_F32 || dtype == LVG_F16, "%s: dtype must be float32 or float16", name);
    LVG_REQUIRE(n >= 1 && c >= 1 && (int64_t)n * c <= 0x7fffffff, "%s: bad n, c", name);
    Axis ax[3];
    for (int a = 0; a < 3; a++) {
        LVG_REQUIRE(in[a] >= 1 && out[a] >= 1 && (filt[a] == 0 || filt[a] == 1), "%s: bad extent or filter flag on axis %d", name, a);
        LVG_REQUIRE(filt[a] || in[a] == out[a], "%s: an unfiltered axis keeps its extent (axis %d)", name, a);
        LVG_REQUIRE(!filt[a] || step[a] == 1 || step[a] == 2, "%s: step must be 1 or 2", name);
        LVG_REQUIRE(!filt[a] || (off[a] >= -8 && off[a] <= 8), "%s: offset out of range", name);
        ax[a] = Axis{filt[a], filt[a] ? step[a] : 1, filt[a] ? off[a] : 0, in[a], out[a]};
    }
    LVG_REQUIRE(!fold || (filt[0] && out[0] % 2 == 0), "%s: fold needs a filtered T axis with an even filtered extent", name);
    const int hout = adj ? in[1] : out[1], wout = adj ? in[2] : out[2];
    const int64_t tiles = (int64_t)((hout + kTH - 1) / kTH) * ((wout + kTW - 1) / kTW);
    LVG_REQUIRE(tiles <= 65535, "%s: plane too large (%lld tiles)", name, (long long)tiles);
    dim3 grid((unsigned)(n * c), (unsigned)tiles);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == LVG_F32) {
        if (adj) fir3d_adjoint_kernel<float><<<grid, kThreads, 0, s>>>((const float*)x, f, (float*)y, c, fold, ax[0], ax[1], ax[2]);
        else fir3d_down_kernel<float><<<grid, kThreads, 0, s>>>((const float*)x, f, (float*)y, c, fold, ax[0], ax[1], ax[2]);
    } else {
        if (adj) fir3d_adjoint_kernel<__half><<<grid, kThreads, 0, s>>>((const __half*)x, f, (__half*)y, c, fold, ax[0], ax[1], ax[2]);
        else fir3d_down_kernel<__half><<<grid, kThreads, 0, s>>>((const __half*)x, f, (__half*)y, c, fold, ax[0], ax[1], ax[2]);
    }
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int lvg_fir3d(const void* x, const float* f, void* y, int dtype, int n, int c, int t_in, int h_in, int w_in, int t_out,
                         int h_out, int w_out, int filt_t, int filt_h, int filt_w, int step_t, int step_h, int step_w, int off_t,
                         int off_h, int off_w, int fold, void* stream)
{
    const int in[3] = {t_in, h_in, w_in}, out[3] = {t_out, h_out, w_out};
    const int filt[3] = {filt_t, filt_h, filt_w}, step[3] = {step_t, step_h, step_w}, off[3] = {off_t, off_h, off_w};
    return fir3d_launch(false, x, f, y, dtype, n, c, in, out, filt, step, off, fold, stream);
}

extern "C" int lvg_fir3d_adjoint(const void* x, const float* f, void* y, int dtype, int n, int c, int t_in, int h_in, int w_in,
                                 int t_out, int h_out, int w_out, int filt_t, int filt_h, int filt_w, int step_t, int step_h,
                                 int step_w, int off_t, int off_h, int off_w, int fold, void* stream)
{
    const int in[3] = {t_in, h_in, w_in}, out[3] = {t_out, h_out, w_out};
    const int filt[3] = {filt_t, filt_h, filt_w}, step[3] = {step_t, step_h, step_w}, off[3] = {off_t, off_h, off_w};
    return fir3d_launch(true, x, f, y, dtype, n, c, in, out, filt, step, off, fold, stream);
}
