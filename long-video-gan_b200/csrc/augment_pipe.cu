// ADA's AugmentPipe (ada_augment.py:115-439) for the super-res step, without imgfilter and cutout, as one affine map per
// sample of x [n][3 * t][h][w] (DESIGN.md 7e):
//
//   y = C[:3,:3] . downsample2d(grid_sample(upsample2d(reflect_pad(x)), affine_grid(theta))) + C[:3,3] + sigma * noise
//
// with the filter Hz_geom (12 taps) read from the device at call time, and without the geometric part y = C x + ... .
// Forward: augment_pipe_fwd_kernel, a CTA per 16 x 16 output tile of one frame's 3 channels; the 42 x 42 v-tile (v = the
// grid-sampled image) is built in shared memory from 7 x 7 windows of the padded x (augment_pipe.cuh), then filtered down.
// Adjoint: augment_pipe_dv_kernel writes dv = D^T (C^T dy) to the workspace; augment_pipe_adjoint_kernel gathers, for each
// x pixel and each of its reflected copies, the v points whose window holds it, weighted with the forward's own function.
// No atomics: both directions are bitwise reproducible.
#include "common.cuh"
#include "augment_pipe.cuh"

namespace lvg {
namespace {

using namespace ap;

constexpr int kThreads = 256;
constexpr int kTile = 16;                   // output tile of the forward
constexpr int kV = 2 * kTile + kTaps - 2;   // v points per tile axis: 2 * 16 + 10

struct Geo {
    int mx0, my0, mx1, my1;
    float th[6];
};

__device__ __forceinline__ Geo load_geo(const float* __restrict__ p) {
    Geo g;
    g.mx0 = __float2int_rn(__ldg(p + 0));
    g.my0 = __float2int_rn(__ldg(p + 1));
    g.mx1 = __float2int_rn(__ldg(p + 2));
    g.my1 = __float2int_rn(__ldg(p + 3));
#pragma unroll
    for (int k = 0; k < 6; k++) g.th[k] = __ldg(p + 4 + k);
    return g;
}

// out_c = sum_c' M[c][c'] in_c' with M = C[:3,:3] (or its transpose)
template <bool TRANSPOSE>
__device__ __forceinline__ void mix(const float* __restrict__ cm, const float (&in)[3], float (&out)[3]) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float m0 = __ldg(cm + (TRANSPOSE ? 0 * 4 + c : c * 4 + 0));
        const float m1 = __ldg(cm + (TRANSPOSE ? 1 * 4 + c : c * 4 + 1));
        const float m2 = __ldg(cm + (TRANSPOSE ? 2 * 4 + c : c * 4 + 2));
        out[c] = __fmaf_rn(m2, in[2], __fmaf_rn(m1, in[1], __fmul_rn(m0, in[0])));
    }
}

// y = C x + offset + sigma noise (forward) or dx = C^T dy (ADJ), per pixel: the map without geometric steps
template <bool ADJ, bool LINEAR>
__global__ void __launch_bounds__(kThreads) augment_pipe_color_kernel(const float* __restrict__ src, const float* __restrict__ par,
                                                                     const float* __restrict__ noise, float* __restrict__ dst, int thw)
{
    const int n = blockIdx.y;
    const int idx = blockIdx.x * kThreads + threadIdx.x;
    if (idx >= thw) return;
    const float* p = par + kNpar * n;
    const int64_t base = (int64_t)n * 3 * thw + idx;
    float in[3], out[3];
#pragma unroll
    for (int c = 0; c < 3; c++) in[c] = __ldg(src + base + (int64_t)c * thw);
    mix<ADJ>(p + 10, in, out);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float v = out[c];
        if (!ADJ && !LINEAR) {
            v = __fadd_rn(v, __ldg(p + 10 + c * 4 + 3));
            if (noise) v = __fadd_rn(v, __fmul_rn(__ldg(noise + base + (int64_t)c * thw), __ldg(p + 22)));
        }
        dst[base + (int64_t)c * thw] = v;
    }
}

template <bool LINEAR>
__global__ void __launch_bounds__(kThreads) augment_pipe_fwd_kernel(const float* __restrict__ x, const float* __restrict__ par,
                                                                   const float* __restrict__ filt, const float* __restrict__ noise,
                                                                   float* __restrict__ y, int t, int h, int w, int tiles_w)
{
    __shared__ float f_s[kTaps];
    __shared__ float vs[3][kV][kV + 1];
    __shared__ float hs[3][kV][kTile + 1];
    const int n = blockIdx.z, tt = blockIdx.y;
    const int oy0 = (blockIdx.x / tiles_w) * kTile, ox0 = (blockIdx.x % tiles_w) * kTile;
    if (threadIdx.x < kTaps) f_s[threadIdx.x] = __ldg(filt + threadIdx.x);
    const float* p = par + kNpar * n;
    const Geo g = load_geo(p);
    const int hp = h + g.my0 + g.my1, wp = w + g.mx0 + g.mx1, hv = 2 * h + 12, wv = 2 * w + 12;
    const int64_t plane = (int64_t)h * w, cstride = (int64_t)t * plane;
    const float* xs = x + (int64_t)n * 3 * cstride + tt * plane;
    __syncthreads();

    // v-tile: v rows 2 * oy0 + 1 + r, columns 2 * ox0 + 1 + q (the ones the down-filter of this output tile reads)
    for (int idx = threadIdx.x; idx < kV * kV; idx += kThreads) {
        const int r = idx / kV, q = idx - r * kV;
        const int vi = 2 * oy0 + 1 + r, vj = 2 * ox0 + 1 + q;
        float acc[3] = {0.f, 0.f, 0.f};
        if (vi < hv && vj < wv) {
            float ix, iy;
            point_coord(g.th, grid_base(vj, wv), grid_base(vi, hv), 2 * wp, 2 * hp, ix, iy);
            const Axis ax = axis_of(ix, 2 * wp), ay = axis_of(iy, 2 * hp);
            if ((ax.a0 != 0.f || ax.a1 != 0.f) && (ay.a0 != 0.f || ay.a1 != 0.f)) {
                float wx[kWin];
                int cx[kWin];
#pragma unroll
                for (int k = 0; k < kWin; k++) {
                    const int i = ax.i0 + k;
                    const bool in = i >= 0 && i < wp;
                    wx[k] = in ? tap(ax, k, f_s) : 0.f;
                    cx[k] = in ? reflect(i, g.mx0, w) : 0;
                }
#pragma unroll 1
                for (int ky = 0; ky < kWin; ky++) {
                    const int i = ay.i0 + ky;
                    if (i < 0 || i >= hp) continue;
                    const float wy = tap(ay, ky, f_s);
                    if (wy == 0.f) continue;
                    const float* row = xs + (int64_t)reflect(i, g.my0, h) * w;
                    float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
                    for (int k = 0; k < kWin; k++) {
#pragma unroll
                        for (int c = 0; c < 3; c++) s[c] = __fmaf_rn(wx[k], __ldg(row + c * cstride + cx[k]), s[c]);
                    }
#pragma unroll
                    for (int c = 0; c < 3; c++) acc[c] = __fmaf_rn(wy, s[c], acc[c]);
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 3; c++) vs[c][r][q] = acc[c];
    }
    __syncthreads();

    // down-filter along W: hs[c][r][o] = sum_k f[k] v[r][2 o + k]
    for (int idx = threadIdx.x; idx < 3 * kV * kTile; idx += kThreads) {
        const int c = idx / (kV * kTile), rem = idx - c * kV * kTile, r = rem / kTile, o = rem - r * kTile;
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kTaps; k++) s = __fmaf_rn(f_s[k], vs[c][r][2 * o + k], s);
        hs[c][r][o] = s;
    }
    __syncthreads();

    // along H, then the colour affine and the noise term
    const int oy = threadIdx.x / kTile, ox = threadIdx.x % kTile;
    if (oy0 + oy >= h || ox0 + ox >= w) return;
    float gv[3], out[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kTaps; k++) s = __fmaf_rn(f_s[k], hs[c][2 * oy + k][ox], s);
        gv[c] = s;
    }
    mix<false>(p + 10, gv, out);
    const int64_t o = (int64_t)n * 3 * cstride + tt * plane + (int64_t)(oy0 + oy) * w + ox0 + ox;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float v = out[c];
        if (!LINEAR) {
            v = __fadd_rn(v, __ldg(p + 10 + c * 4 + 3));
            if (noise) v = __fadd_rn(v, __fmul_rn(__ldg(noise + o + c * cstride), __ldg(p + 22)));
        }
        y[o + c * cstride] = v;
    }
}

// dv = D^T (C^T dy) for one v point of one frame, 3 channels: g[o] = sum_k f[k] v[2 o + 1 + k] per axis
__global__ void __launch_bounds__(kThreads) augment_pipe_dv_kernel(const float* __restrict__ dy, const float* __restrict__ par,
                                                                  const float* __restrict__ filt, float* __restrict__ dv, int t, int h,
                                                                  int w)
{
    const int n = blockIdx.z, tt = blockIdx.y;
    const int hv = 2 * h + 12, wv = 2 * w + 12;
    const int idx = blockIdx.x * kThreads + threadIdx.x;
    if (idx >= hv * wv) return;
    const int vi = idx / wv, vj = idx - vi * wv;
    const int64_t plane = (int64_t)h * w, cstride = (int64_t)t * plane;
    const float* ds = dy + (int64_t)n * 3 * cstride + tt * plane;
    // o with 0 <= v - 1 - 2 o < 12 and 0 <= o < size
    const int oy_lo = max(0, floor_div2(vi - 11)), oy_hi = min(h - 1, floor_div2(vi - 1));
    const int ox_lo = max(0, floor_div2(vj - 11)), ox_hi = min(w - 1, floor_div2(vj - 1));
    float acc[3] = {0.f, 0.f, 0.f};
    for (int oy = oy_lo; oy <= oy_hi; oy++) {
        const float fy = __ldg(filt + vi - 1 - 2 * oy);
        float s[3] = {0.f, 0.f, 0.f};
        for (int ox = ox_lo; ox <= ox_hi; ox++) {
            const float fx = __ldg(filt + vj - 1 - 2 * ox);
#pragma unroll
            for (int c = 0; c < 3; c++) s[c] = __fmaf_rn(fx, __ldg(ds + c * cstride + (int64_t)oy * w + ox), s[c]);
        }
#pragma unroll
        for (int c = 0; c < 3; c++) acc[c] = __fmaf_rn(fy, s[c], acc[c]);
    }
    float out[3];
    mix<true>(par + kNpar * n + 10, acc, out);
    const int64_t vplane = (int64_t)hv * wv;
    float* o = dv + ((int64_t)n * 3 * t + tt) * vplane + idx;
#pragma unroll
    for (int c = 0; c < 3; c++) o[c * t * vplane] = out[c];
}

// dx of one x pixel, 3 channels: the transpose of the forward's v-tile sum, point by point over the enumeration boxes
__global__ void __launch_bounds__(kThreads) augment_pipe_adjoint_kernel(const float* __restrict__ dv, const float* __restrict__ par,
                                                                       const float* __restrict__ filt, float* __restrict__ dx, int t,
                                                                       int h, int w)
{
    __shared__ float f_s[kTaps];
    const int n = blockIdx.z, tt = blockIdx.y;
    if (threadIdx.x < kTaps) f_s[threadIdx.x] = __ldg(filt + threadIdx.x);
    __syncthreads();
    const int idx = blockIdx.x * kThreads + threadIdx.x;
    if (idx >= h * w) return;
    const int yy = idx / w, xx = idx - yy * w;
    const Geo g = load_geo(par + kNpar * n);
    const int hp = h + g.my0 + g.my1, wp = w + g.mx0 + g.mx1, hv = 2 * h + 12, wv = 2 * w + 12;
    const int lux = 2 * wp, luy = 2 * hp;
    const int64_t vplane = (int64_t)hv * wv, vcs = (int64_t)t * vplane;
    const float* ds = dv + ((int64_t)n * 3 * t + tt) * vplane;
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
    for (int a = 0; a < 3; a++) {
        const int py = copy_at(yy, g.my0, g.my1, h, a);
        if (py < 0) continue;
#pragma unroll 1
        for (int b = 0; b < 3; b++) {
            const int px = copy_at(xx, g.mx0, g.mx1, w, b);
            if (px < 0) continue;
            const Box box = box_rows(g.th, px, py, lux, luy, hv);
            for (int vi = box.vi_lo; vi <= box.vi_hi; vi++) {
                const float yb = grid_base(vi, hv);
                int j_lo, j_hi;
                if (!box_cols(g.th, box, yb, wv, j_lo, j_hi)) continue;
                for (int vj = j_lo; vj <= j_hi; vj++) {
                    float ix, iy;
                    point_coord(g.th, grid_base(vj, wv), yb, lux, luy, ix, iy);
                    const Axis ax = axis_of(ix, lux);
                    const int kx = px - ax.i0;
                    if (kx < 0 || kx >= kWin) continue;
                    const Axis ay = axis_of(iy, luy);
                    const int ky = py - ay.i0;
                    if (ky < 0 || ky >= kWin) continue;
                    const float wt = __fmul_rn(tap(ay, ky, f_s), tap(ax, kx, f_s));
                    if (wt == 0.f) continue;
                    const float* d = ds + (int64_t)vi * wv + vj;
#pragma unroll
                    for (int c = 0; c < 3; c++) acc[c] = __fmaf_rn(wt, __ldg(d + c * vcs), acc[c]);
                }
            }
        }
    }
    const int64_t plane = (int64_t)h * w, cstride = (int64_t)t * plane;
    float* o = dx + (int64_t)n * 3 * cstride + tt * plane + idx;
#pragma unroll
    for (int c = 0; c < 3; c++) o[c * cstride] = acc[c];
}

bool shape_ok(int n, int c, int t, int h, int w) {
    return n >= 1 && n <= 65535 && c == 3 && t >= 1 && t <= 65535 && h >= 1 && w >= 1 &&
           (int64_t)(2 * (int64_t)h + 12) * (2 * (int64_t)w + 12) < ((int64_t)1 << 31) && (int64_t)c * t * h * w < ((int64_t)1 << 31);
}

int64_t workspace_bytes(int n, int c, int t, int h, int w, int flags) {
    if (!(flags & LVG_AUGMENT_PIPE_GEOM)) return 0;
    return (int64_t)n * c * t * (2 * (int64_t)h + 12) * (2 * (int64_t)w + 12) * (int64_t)sizeof(float);
}

int augment_pipe_launch(bool adj, const float* src, const float* par, const float* filt, int ntaps, const float* noise, float* dst,
                        void* ws, int n, int c, int t, int h, int w, int flags, void* stream)
{
    const char* name = adj ? "augment_pipe_adjoint" : "augment_pipe";
    if (c != 3 || ntaps != kTaps) return LVG_UNSUPPORTED;
    LVG_REQUIRE((flags & ~(LVG_AUGMENT_PIPE_GEOM | LVG_AUGMENT_PIPE_LINEAR)) == 0, "%s: unknown flags %d", name, flags);
    const bool geom = flags & LVG_AUGMENT_PIPE_GEOM, linear = flags & LVG_AUGMENT_PIPE_LINEAR;
    LVG_REQUIRE(src && par && dst && (filt || !geom) && (ws || !adj || !geom), "%s: x, params, filter, y and workspace must not be NULL",
                name);
    LVG_REQUIRE(shape_ok(n, c, t, h, w), "%s: bad shape n=%d c=%d t=%d h=%d w=%d", name, n, c, t, h, w);
    cudaStream_t s = (cudaStream_t)stream;
    const int thw = t * h * w;
    if (!geom) {
        const dim3 grid((unsigned)((thw + kThreads - 1) / kThreads), n);
        if (adj) augment_pipe_color_kernel<true, true><<<grid, kThreads, 0, s>>>(src, par, nullptr, dst, thw);
        else if (linear) augment_pipe_color_kernel<false, true><<<grid, kThreads, 0, s>>>(src, par, nullptr, dst, thw);
        else augment_pipe_color_kernel<false, false><<<grid, kThreads, 0, s>>>(src, par, noise, dst, thw);
    } else if (!adj) {
        const int tiles_w = (w + kTile - 1) / kTile, tiles_h = (h + kTile - 1) / kTile;
        const dim3 grid((unsigned)(tiles_w * tiles_h), t, n);
        if (linear) augment_pipe_fwd_kernel<true><<<grid, kThreads, 0, s>>>(src, par, filt, nullptr, dst, t, h, w, tiles_w);
        else augment_pipe_fwd_kernel<false><<<grid, kThreads, 0, s>>>(src, par, filt, noise, dst, t, h, w, tiles_w);
    } else {
        float* dv = (float*)ws;
        const int hvwv = (2 * h + 12) * (2 * w + 12);
        augment_pipe_dv_kernel<<<dim3((unsigned)((hvwv + kThreads - 1) / kThreads), t, n), kThreads, 0, s>>>(src, par, filt, dv, t, h, w);
        LVG_LAUNCH_CHECK();
        augment_pipe_adjoint_kernel<<<dim3((unsigned)((h * w + kThreads - 1) / kThreads), t, n), kThreads, 0, s>>>(dv, par, filt, dst, t, h, w);
    }
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_augment_pipe_workspace(int n, int c, int t, int h, int w, int flags)
{
    if (!shape_ok(n, c, t, h, w)) return LVG_UNSUPPORTED;
    return workspace_bytes(n, c, t, h, w, flags);
}

extern "C" int lvg_augment_pipe(const float* x, const float* params, const float* filter, int ntaps, const float* noise, float* y, int n,
                                int c, int t, int h, int w, int flags, void* stream)
{
    return augment_pipe_launch(false, x, params, filter, ntaps, noise, y, nullptr, n, c, t, h, w, flags, stream);
}

extern "C" int lvg_augment_pipe_adjoint(const float* dy, const float* params, const float* filter, int ntaps, float* dx, void* workspace,
                                        int n, int c, int t, int h, int w, int flags, void* stream)
{
    return augment_pipe_launch(true, dy, params, filter, ntaps, nullptr, dx, workspace, n, c, t, h, w, flags | LVG_AUGMENT_PIPE_LINEAR,
                               stream);
}
