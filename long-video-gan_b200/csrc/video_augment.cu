// Input augmentation of the low-res discriminator (LowResVideoGAN.run_D, video_gan_lres.py:237-266): DiffAugment's
// color, translation and cutout steps (diff_augment.py) and the temporal-scale augmentation, as one affine map per sample
//
//   y[c][t][h][w] = mask(h, w) * sum_k lambda_k(t) * z[c][tap_k(t)][h + dh][w + dw],   z = a x + b m + (1 - kappa) mu + beta
//
// with a = kappa sigma, b = kappa (1 - sigma), m the per-pixel channel mean and mu the per-sample mean of x (DESIGN.md 7d).
// mask is zero outside the frame after translation and inside the cutout rectangle; the two temporal taps are
// F.interpolate(align_corners=False)'s, in its fp32 index arithmetic, for u = t + off in [0, L) and zero elsewhere.
//
// Forward: video_augment_reduce_kernel<0> writes per-CTA partial sums of x; the gather kernel folds them in a fixed order
// (every CTA the same way) and each thread produces one output pixel with all C channels, reading its <= 2 source frames.
// Adjoint: video_augment_reduce_kernel<1> sums dy over the positions whose taps land inside x (the sum of g, the adjoint of
// the gather, without forming g), then each thread gathers g for one input pixel by walking the output frames whose taps
// reach its frame, with the forward's own index arithmetic, and applies the transposed color step. No atomics: both
// directions are bitwise reproducible.
#include "common.cuh"

namespace lvg {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxParts = 256;          // partial sums per sample (<= kThreads: the fold loads one per thread)
constexpr int kElemsPerPart = 8192;

struct Par {
    float beta, sigma, kappa;
    int dh, dw, r0, r1, c0, c1;
    float r;
    int len, off;
};

__device__ __forceinline__ Par load_par(const float* __restrict__ p) {
    Par q;
    q.beta = __ldg(p + 0);
    q.sigma = __ldg(p + 1);
    q.kappa = __ldg(p + 2);
    q.dh = __float2int_rn(__ldg(p + 3));
    q.dw = __float2int_rn(__ldg(p + 4));
    q.r0 = __float2int_rn(__ldg(p + 5));
    q.r1 = __float2int_rn(__ldg(p + 6));
    q.c0 = __float2int_rn(__ldg(p + 7));
    q.c1 = __float2int_rn(__ldg(p + 8));
    q.r = __ldg(p + 9);
    q.len = __float2int_rn(__ldg(p + 10));
    q.off = __float2int_rn(__ldg(p + 11));
    return q;
}

// output pixel (oh, ow) reads input pixel (oh + dh, ow + dw) and is not cut out
__device__ __forceinline__ bool pixel_kept(const Par& p, int oh, int ow, int h, int w) {
    const int sh = oh + p.dh, sw = ow + p.dw;
    return sh >= 0 && sh < h && sw >= 0 && sw < w && !(oh >= p.r0 && oh <= p.r1 && ow >= p.c0 && ow <= p.c1);
}

// first temporal tap of clip frame u (0 <= u < L) and its neighbour's weight, as upsample_linear's align_corners=False
// source index: src = max(0, r (u + 0.5) - 0.5), h1 = floor(src), lambda1 = src - h1, second tap min(h1 + 1, T - 1)
__device__ __forceinline__ int tap_of(float r, int u, int t_in, float& l1) {
    const float src = fmaxf(__fmaf_rn(r, (float)u + 0.5f, -0.5f), 0.f);
    const int h1 = min((int)src, t_in - 1);
    l1 = src - (float)h1;
    return h1;
}

// sum over the CTA in a fixed order; the result is valid in thread 0
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < kThreads / 32 ? red[lane] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    }
    return v;
}

// the per-sample mean from the reduce kernel's partial sums, identical in every CTA
__device__ __forceinline__ float fold_mean(const float* __restrict__ parts, int nparts, float count) {
    __shared__ float red[kThreads / 32];
    __shared__ float total;
    const float s = block_sum(threadIdx.x < nparts ? parts[threadIdx.x] : 0.f, red);
    if (threadIdx.x == 0) total = s / count;
    __syncthreads();
    return total;
}

// MODE 0: partial sums of x over each sample. MODE 1: partial sums of dy over the output positions that read x
// (u inside [0, L), pixel kept) -- the sum of the gather's adjoint, since the two tap weights of a frame sum to one.
template <int MODE>
__global__ void __launch_bounds__(kThreads) video_augment_reduce_kernel(const float* __restrict__ src, const float* __restrict__ par,
                                                                       float* __restrict__ parts, int nparts, int c, int t, int h, int w)
{
    __shared__ float red[kThreads / 32];
    const int n = blockIdx.y;
    const int plane = h * w, frames = t * plane, count = c * frames;       // < 2^31 (shape_ok)
    const int chunk = (count + nparts - 1) / nparts;
    const int begin = blockIdx.x * chunk, end = min(count, begin + chunk);
    const float* s = src + (int64_t)n * count;
    Par p{};
    if (MODE == 1) p = load_par(par + 12 * n);
    float acc = 0.f;
    for (int i = begin + threadIdx.x; i < end; i += kThreads) {
        if (MODE == 1) {
            const int rem = i % frames;
            const int tt = rem / plane, pix = rem - tt * plane, oh = pix / w, ow = pix - oh * w;
            const int u = tt + p.off;
            if (u < 0 || u >= p.len || !pixel_kept(p, oh, ow, h, w)) continue;
        }
        acc += __ldg(s + i);
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) parts[n * nparts + blockIdx.x] = acc;
}

template <int C, bool LINEAR>
__global__ void __launch_bounds__(kThreads) video_augment_fwd_kernel(const float* __restrict__ x, const float* __restrict__ par,
                                                                    const float* __restrict__ parts, int nparts, float* __restrict__ y,
                                                                    int t_in, int h, int w, int t_out)
{
    const int n = blockIdx.y;
    const int64_t plane = (int64_t)h * w;
    const float mu = fold_mean(parts + n * nparts, nparts, (float)((double)C * t_in * plane));
    const int64_t idx = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (idx >= t_out * plane) return;
    const Par p = load_par(par + 12 * n);
    const int t = (int)(idx / plane), pix = (int)(idx - t * plane), oh = pix / w, ow = pix - oh * w;
    float acc[C];
#pragma unroll
    for (int ci = 0; ci < C; ci++) acc[ci] = 0.f;
    const int u = t + p.off;
    if (u >= 0 && u < p.len && pixel_kept(p, oh, ow, h, w)) {
        float l1;
        const int f1 = tap_of(p.r, u, t_in, l1), f2 = min(f1 + 1, t_in - 1);
        const float a = p.kappa * p.sigma, b = p.kappa * (1.f - p.sigma), c0 = (1.f - p.kappa) * mu + (LINEAR ? 0.f : p.beta);
        const float* xs = x + (int64_t)n * C * t_in * plane + (int64_t)(oh + p.dh) * w + (ow + p.dw);
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const int f = k == 0 ? f1 : f2;
            const float wk = k == 0 ? 1.f - l1 : l1;
            float v[C], m = 0.f;
#pragma unroll
            for (int ci = 0; ci < C; ci++) {
                v[ci] = __ldg(xs + ((int64_t)ci * t_in + f) * plane);
                m += v[ci];
            }
            m = m / (float)C;
#pragma unroll
            for (int ci = 0; ci < C; ci++) acc[ci] = __fmaf_rn(wk, __fmaf_rn(a, v[ci], __fmaf_rn(b, m, c0)), acc[ci]);
        }
    }
    float* ys = y + (int64_t)n * C * t_out * plane + idx;
#pragma unroll
    for (int ci = 0; ci < C; ci++) ys[(int64_t)ci * t_out * plane] = acc[ci];
}

template <int C>
__global__ void __launch_bounds__(kThreads) video_augment_adjoint_kernel(const float* __restrict__ dy, const float* __restrict__ par,
                                                                        const float* __restrict__ parts, int nparts, float* __restrict__ dx,
                                                                        int t_in, int h, int w, int t_out)
{
    const int n = blockIdx.y;
    const int64_t plane = (int64_t)h * w;
    const float gbar = fold_mean(parts + n * nparts, nparts, (float)((double)C * t_in * plane));
    const int64_t idx = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (idx >= t_in * plane) return;
    const Par p = load_par(par + 12 * n);
    const int j = (int)(idx / plane), pix = (int)(idx - j * plane), ih = pix / w, iw = pix - ih * w;
    const int oh = ih - p.dh, ow = iw - p.dw;                  // the output pixel that reads this input pixel
    float g[C];
#pragma unroll
    for (int ci = 0; ci < C; ci++) g[ci] = 0.f;
    if (oh >= 0 && oh < h && ow >= 0 && ow < w && pixel_kept(p, oh, ow, h, w)) {
        // clip frames u whose first tap is j - 1 or j: a contiguous range, since the tap is non-decreasing in u
        const int u_lo = max(0, p.off), u_hi = min(p.len, t_out + p.off);
        float l1;
        int u = max(u_lo, (int)(((float)j - 0.5f) / p.r - 0.5f) - 2);
        while (u > u_lo && tap_of(p.r, u, t_in, l1) >= j - 1) u--;
        const float* ds = dy + (int64_t)n * C * t_out * plane + (int64_t)oh * w + ow;
        for (; u < u_hi; u++) {
            const int f1 = tap_of(p.r, u, t_in, l1);
            if (f1 > j) break;
            const int f2 = min(f1 + 1, t_in - 1);
            const float wt = (f1 == j ? 1.f - l1 : 0.f) + (f2 == j ? l1 : 0.f);
            if (f1 < j - 1 || wt == 0.f) continue;
            const int t = u - p.off;
#pragma unroll
            for (int ci = 0; ci < C; ci++) g[ci] = __fmaf_rn(wt, __ldg(ds + ((int64_t)ci * t_out + t) * plane), g[ci]);
        }
    }
    float gm = 0.f;
#pragma unroll
    for (int ci = 0; ci < C; ci++) gm += g[ci];
    gm = gm / (float)C;
    const float a = p.kappa * p.sigma, b = p.kappa * (1.f - p.sigma), c0 = (1.f - p.kappa) * gbar;
    float* xs = dx + (int64_t)n * C * t_in * plane + idx;
#pragma unroll
    for (int ci = 0; ci < C; ci++) xs[(int64_t)ci * t_in * plane] = __fmaf_rn(a, g[ci], __fmaf_rn(b, gm, c0));
}

int num_parts(int c, int t, int h, int w) {
    const int64_t parts = ((int64_t)c * t * h * w + kElemsPerPart - 1) / kElemsPerPart;
    return parts < 1 ? 1 : parts > kMaxParts ? kMaxParts : (int)parts;
}

bool shape_ok(int n, int c, int t_in, int h, int w, int t_out) {
    return n >= 1 && n <= 65535 && c >= 1 && t_in >= 1 && h >= 1 && w >= 1 && t_out >= 1 &&
           (int64_t)c * max(t_in, t_out) * h * w < ((int64_t)1 << 31);
}

template <int C>
void launch(bool adj, const float* src, const float* par, float* dst, float* parts, int n, int t_in, int h, int w, int t_out,
            bool linear, cudaStream_t s)
{
    const int t_src = adj ? t_out : t_in, t_dst = adj ? t_in : t_out;
    const int np = num_parts(C, t_src, h, w);
    const dim3 rgrid(np, n), ggrid((unsigned)(((int64_t)t_dst * h * w + kThreads - 1) / kThreads), n);
    if (adj) {
        video_augment_reduce_kernel<1><<<rgrid, kThreads, 0, s>>>(src, par, parts, np, C, t_out, h, w);
        video_augment_adjoint_kernel<C><<<ggrid, kThreads, 0, s>>>(src, par, parts, np, dst, t_in, h, w, t_out);
    } else {
        video_augment_reduce_kernel<0><<<rgrid, kThreads, 0, s>>>(src, par, parts, np, C, t_in, h, w);
        if (linear) video_augment_fwd_kernel<C, true><<<ggrid, kThreads, 0, s>>>(src, par, parts, np, dst, t_in, h, w, t_out);
        else video_augment_fwd_kernel<C, false><<<ggrid, kThreads, 0, s>>>(src, par, parts, np, dst, t_in, h, w, t_out);
    }
}

int video_augment_launch(bool adj, const float* src, const float* par, float* dst, void* ws, int n, int c, int t_in, int h, int w,
                         int t_out, int flags, void* stream)
{
    const char* name = adj ? "video_augment_adjoint" : "video_augment";
    if (c > 4) return LVG_UNSUPPORTED;
    LVG_REQUIRE(src && par && dst && ws, "%s: x, params, y and workspace must not be NULL", name);
    LVG_REQUIRE(shape_ok(n, c, t_in, h, w, t_out), "%s: bad shape n=%d c=%d t_in=%d h=%d w=%d t_out=%d", name, n, c, t_in, h, w, t_out);
    LVG_REQUIRE((flags & ~LVG_VIDEO_AUGMENT_LINEAR) == 0, "%s: unknown flags %d", name, flags);
    const bool linear = flags & LVG_VIDEO_AUGMENT_LINEAR;
    cudaStream_t s = (cudaStream_t)stream;
    float* parts = (float*)ws;
    switch (c) {
        case 1: launch<1>(adj, src, par, dst, parts, n, t_in, h, w, t_out, linear, s); break;
        case 2: launch<2>(adj, src, par, dst, parts, n, t_in, h, w, t_out, linear, s); break;
        case 3: launch<3>(adj, src, par, dst, parts, n, t_in, h, w, t_out, linear, s); break;
        default: launch<4>(adj, src, par, dst, parts, n, t_in, h, w, t_out, linear, s); break;
    }
    count_launch();                          // two kernels per call
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_video_augment_workspace(int n, int c, int t_in, int h, int w, int t_out)
{
    if (c > 4 || !shape_ok(n, c, t_in, h, w, t_out)) return LVG_UNSUPPORTED;
    return (int64_t)n * max(num_parts(c, t_in, h, w), num_parts(c, t_out, h, w)) * (int64_t)sizeof(float);
}

extern "C" int lvg_video_augment(const float* x, const float* params, float* y, void* workspace, int n, int c, int t_in, int h,
                                 int w, int t_out, int flags, void* stream)
{
    return video_augment_launch(false, x, params, y, workspace, n, c, t_in, h, w, t_out, flags, stream);
}

extern "C" int lvg_video_augment_adjoint(const float* dy, const float* params, float* dx, void* workspace, int n, int c, int t_in,
                                         int h, int w, int t_out, void* stream)
{
    return video_augment_launch(true, dy, params, dx, workspace, n, c, t_in, h, w, t_out, 0, stream);
}
