// The super-res generator's ToRGB layer (DESIGN.md 7k) as one pass over its input:
//
//   z = cat(x_prev, cond(lr)).to(dtype)                        lvg_sres_cond's layer input, never stored
//   u = conv1x1(r(a (.) z), w)                                 w = dtype(wn) [3][cin], a [n t][cin]
//   y = dtype(clamp(dtype(u) + b, +-clamp))                    filtered_lrelu's 1x1 path with gain 1 and slope 1
//
// r() is the rounding of the convolution engine's re-tiling pass (conv_pack_act_kernel / conv_pack_cond_kernel): fp16
// layers round a z to fp16, fp32 layers keep it in fp32. Every product is accumulated in fp32 on the CUDA cores: a 3-row
// output does not fill a tensor-core tile, and the layer moves 128 input channels per 3 output channels, so it is bound by
// HBM. A CTA owns a tile of output rows of one sample; each thread owns a run of 8 output pixels and keeps the 3 x 8
// accumulators in registers. x_prev is read with 16-byte loads when every row starts on a 16-byte boundary (the width a
// multiple of 8 and x_prev, dy and dx 16-byte aligned), with scalar loads otherwise. The conditioning channels are
// evaluated in place by the layer's plan with the tap tables and both FIR passes of sres_cond.cuh (the vertical pass of the
// tile staged in shared memory), so they round to the bits lvg_sres_cond writes.
//
// The forward optionally writes one byte per pixel: bit o set where output o was clamped (|dtype(u) + b| > clamp), the
// mask filtered_lrelu's gradient applies. The backward reads x_prev and dy once and writes dx_prev once:
//   dy' = dy where not clamped, else 0
//   dx' = dtype(w^T dy')                          per pixel, as the engine's input gradient stores it
//   dx_prev = x_dtype(dtype(a dx'))               the x_prev channels (the cast of z's gradient)
//   da[n t][c] = sum_p dx' z                      modconv_rowdot's dot of dx' with dtype(z)
//   G[n t][o][c] = sum_p dy' r(a z),  dw = dtype(sum_nt G),  db = dtype(sum dy')
// Each CTA writes its sums to one partial; two small kernels fold them in a fixed order (no atomics: every gradient is
// bitwise reproducible).
#include <algorithm>

#include "common.cuh"
#include "sres_cond.cuh"

namespace lvg {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPix = 8;                       // output pixels per thread
constexpr int kCout = 3;
constexpr int kTilePix = kThreads * kPix;     // output pixels per CTA when the width allows
constexpr int kMaxSmem = 100 * 1024;          // two CTAs per SM
constexpr int kMaxCin = 1024;

struct TorgbParams {
    const void* x;                            // x_prev [np][c][h][w] (TX)
    const float* lr;
    const void* w;                            // [3][cin] (T)
    const float* a;                           // [np][cin]
    const void* b;                            // [3] (T)
    void* y;                                  // [np][3][h][w] (T)
    unsigned char* mask;                      // [np][h][w] or nullptr
    const void* dy;                           // [np][3][h][w] (T)
    void* dx;                                 // x_prev's gradient (TX) or nullptr
    float* part;                              // [ctas][4 cin + 3]
    int64_t s_n, s_c, s_t, s_h, s_w;          // element strides of lr
    int t, c, cin, cc, window;
    int rows, row_tiles;
    int vec;
    float clamp;
    sres::Axis ah, aw;
};

template <class T> __device__ __forceinline__ float rnd(float v);
template <> __device__ __forceinline__ float rnd<float>(float v) { return v; }
template <> __device__ __forceinline__ float rnd<__half>(float v) { return __half2float(__float2half_rn(v)); }

// kPix consecutive elements at p (n of them valid when not vec)
template <class T>
__device__ __forceinline__ void load_run(const T* __restrict__ p, bool vec, int n, float (&v)[kPix])
{
    if (vec) {
        if constexpr (sizeof(T) == 2) {
            float f[8];
            unpack<__half>(load_pack(reinterpret_cast<const __half*>(p)), f);
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = f[k];
        } else {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                float f[4];
                unpack<float>(load_pack(reinterpret_cast<const float*>(p) + 4 * h), f);
#pragma unroll
                for (int k = 0; k < 4; k++) v[4 * h + k] = f[k];
            }
        }
    } else {
#pragma unroll
        for (int k = 0; k < kPix; k++) v[k] = k < n ? to_acc(__ldg(p + k)) : 0.f;
    }
}

template <class T>
__device__ __forceinline__ void store_run(T* __restrict__ p, bool vec, int n, const float (&v)[kPix])
{
    if (vec) {
        if constexpr (sizeof(T) == 2) {
            store_pack(reinterpret_cast<__half*>(p), pack<__half>(v));
        } else {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const float f[4] = {v[4 * h], v[4 * h + 1], v[4 * h + 2], v[4 * h + 3]};
                store_pack(reinterpret_cast<float*>(p) + 4 * h, pack<float>(f));
            }
        }
    } else {
#pragma unroll
        for (int k = 0; k < kPix; k++)
            if (k < n) p[k] = from_acc<T>(v[k]);
    }
}

// shared memory of a tile: [vertical pass cc][rows][w_lr] [row taps rows][nth] x2 [column taps w_out][ntw] x2
// [w as fp32 3][cin] [a cin] and, in the backward, [per-warp sums kWarps][4 cin + 3]
struct TileSmem {
    int64_t inter, wh, sh, ww, sw, wf, af, red, total;
};
__host__ __device__ inline TileSmem tile_smem(int cc, int rows, int wl, int nth, int wout, int ntw, int cin, bool bwd)
{
    TileSmem s;
    s.inter = 0;
    s.wh = s.inter + (int64_t)cc * rows * wl;
    s.sh = s.wh + (int64_t)rows * nth;
    s.ww = s.sh + (int64_t)rows * nth;
    s.sw = s.ww + (int64_t)wout * ntw;
    s.wf = s.sw + (int64_t)wout * ntw;
    s.af = s.wf + (int64_t)kCout * cin;
    s.red = s.af + cin;
    s.total = (s.red + (bwd ? (int64_t)kWarps * (4 * cin + kCout) : 0)) * 4;
    return s;
}

// The tile every thread of both kernels works on: its sample, rows, the pixel run of this thread (r, i per pixel) and the
// shared-memory prologue (tap tables, the vertical pass of the conditioning channels, w and a of the sample).
template <class T>
struct Tile {
    float* smem;
    TileSmem L;
    int64_t np, pix0;                          // sample, first pixel of the tile in the plane
    int n, t, r0, rows, npix;
    __device__ Tile(const TorgbParams& p, float* s, bool bwd) : smem(s)
    {
        L = tile_smem(p.cc, p.rows, p.aw.len, p.ah.nt, p.aw.out, p.aw.nt, p.cin, bwd);
        const int tile = (int)(blockIdx.x % p.row_tiles);
        np = blockIdx.x / p.row_tiles;
        n = (int)(np / p.t);
        t = (int)(np % p.t);
        r0 = tile * p.rows;
        rows = min(p.rows, p.ah.out - r0);
        npix = rows * p.aw.out;
        pix0 = (int64_t)r0 * p.aw.out;

        const int nth = p.ah.nt, ntw = p.aw.nt, wl = p.aw.len;
        float* wh = smem + L.wh;
        int* sh = reinterpret_cast<int*>(smem + L.sh);
        float* ww = smem + L.ww;
        int* sw = reinterpret_cast<int*>(smem + L.sw);
        if (p.cc > 0) {
            for (int r = threadIdx.x; r < rows; r += kThreads) sres::axis_taps(p.ah, r0 + r, sh + r * nth, wh + r * nth);
            for (int i = threadIdx.x; i < p.aw.out; i += kThreads) sres::axis_taps(p.aw, i, sw + i * ntw, ww + i * ntw);
        }
        const T* w = reinterpret_cast<const T*>(p.w);
        for (int k = threadIdx.x; k < kCout * p.cin; k += kThreads) smem[L.wf + k] = to_acc(__ldg(w + k));
        for (int k = threadIdx.x; k < p.cin; k += kThreads) smem[L.af + k] = __ldg(p.a + np * p.cin + k);
        __syncthreads();
        // channel j at j * p.rows * wl (the full tile's stride, which cond_run reads), rows below `rows` in a last tile
        const int plane = rows * wl;
        for (int idx = threadIdx.x; idx < p.cc * plane; idx += kThreads) {
            const int j = idx / plane, r = (idx % plane) / wl, x = idx % wl;
            const int k = j / p.window, s = j % p.window;
            const float* __restrict__ src = p.lr + n * p.s_n + k * p.s_c + (int64_t)(t + s) * p.s_t;
            smem[L.inter + ((int64_t)j * p.rows + r) * wl + x] =
                sres::vertical_tap_sum(src, p.s_h, p.s_w, x, wh + r * nth, sh + r * nth, nth);
        }
        __syncthreads();
    }

    // conditioning channel j at the pixels of a run: the horizontal pass, rounded to the layer dtype as lvg_sres_cond does
    __device__ __forceinline__ void cond_run(const TorgbParams& p, int j, const int (&roff)[kPix], const int (&toff)[kPix], int nv,
                                             float (&z)[kPix]) const
    {
        const float* inter = smem + L.inter + (int64_t)j * p.rows * p.aw.len;
        const float* ww = smem + L.ww;
        const int* sw = reinterpret_cast<const int*>(smem + L.sw);
#pragma unroll
        for (int k = 0; k < kPix; k++)
            z[k] = k < nv ? rnd<T>(sres::horizontal_tap_sum(inter + roff[k], ww + toff[k], sw + toff[k], p.aw.nt)) : 0.f;
    }
};

// offsets of a run's pixels into the vertical pass (row) and the column tap tables
__device__ __forceinline__ void run_offsets(const TorgbParams& p, int q0, int (&roff)[kPix], int (&toff)[kPix])
{
#pragma unroll
    for (int k = 0; k < kPix; k++) {
        const int q = q0 + k, r = q / p.aw.out, i = q - r * p.aw.out;
        roff[k] = r * p.aw.len;
        toff[k] = i * p.aw.nt;
    }
}

template <class TX, class T>
__global__ void __launch_bounds__(kThreads, 2) sres_torgb_fprop_kernel(const TorgbParams p)
{
    extern __shared__ __align__(16) float smem_f[];
    const Tile<T> tl(p, smem_f, false);
    const int64_t hw = (int64_t)p.ah.out * p.aw.out;
    const bool vec = p.vec != 0;
    const float* wf = smem_f + tl.L.wf;
    const float* af = smem_f + tl.L.af;
    const TX* __restrict__ xs = reinterpret_cast<const TX*>(p.x) + tl.np * p.c * hw;
    const T* bs = reinterpret_cast<const T*>(p.b);
    float bias[kCout];
#pragma unroll
    for (int o = 0; o < kCout; o++) bias[o] = to_acc(__ldg(bs + o));

    for (int q0 = threadIdx.x * kPix; q0 < tl.npix; q0 += kThreads * kPix) {
        const int nv = min(kPix, tl.npix - q0);
        const int64_t pix = tl.pix0 + q0;
        // the x_prev channels in two interleaved sums (even / odd channel), added before the conditioning channels:
        // half the depth of one running sum, so fp32 layers stay within 2^-22 of sum |w a z|
        float acc[kCout][kPix], acc1[kCout][kPix];
#pragma unroll
        for (int o = 0; o < kCout; o++)
#pragma unroll
            for (int k = 0; k < kPix; k++) acc[o][k] = acc1[o][k] = 0.f;
        for (int ch = 0; ch < p.c; ch += 2) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                if (ch + h >= p.c) break;
                float v[kPix];
                load_run(xs + (ch + h) * hw + pix, vec, nv, v);
                const float a = af[ch + h], w0 = wf[ch + h], w1 = wf[p.cin + ch + h], w2 = wf[2 * p.cin + ch + h];
                float (&s)[kCout][kPix] = h ? acc1 : acc;
#pragma unroll
                for (int k = 0; k < kPix; k++) {
                    const float az = rnd<T>(rnd<T>(v[k]) * a);
                    s[0][k] = fmaf(w0, az, s[0][k]);
                    s[1][k] = fmaf(w1, az, s[1][k]);
                    s[2][k] = fmaf(w2, az, s[2][k]);
                }
            }
        }
#pragma unroll
        for (int o = 0; o < kCout; o++)
#pragma unroll
            for (int k = 0; k < kPix; k++) acc[o][k] += acc1[o][k];
        if (p.cc > 0) {
            int roff[kPix], toff[kPix];
            run_offsets(p, q0, roff, toff);
            for (int j = 0; j < p.cc; j++) {
                float z[kPix];
                tl.cond_run(p, j, roff, toff, nv, z);
                const int ch = p.c + j;
                const float a = af[ch], w0 = wf[ch], w1 = wf[p.cin + ch], w2 = wf[2 * p.cin + ch];
#pragma unroll
                for (int k = 0; k < kPix; k++) {
                    const float az = rnd<T>(z[k] * a);
                    acc[0][k] = fmaf(w0, az, acc[0][k]);
                    acc[1][k] = fmaf(w1, az, acc[1][k]);
                    acc[2][k] = fmaf(w2, az, acc[2][k]);
                }
            }
        }
        unsigned code[kPix];
#pragma unroll
        for (int k = 0; k < kPix; k++) code[k] = 0;
        T* ys = reinterpret_cast<T*>(p.y) + tl.np * kCout * hw + pix;
#pragma unroll
        for (int o = 0; o < kCout; o++) {
            float out[kPix];
#pragma unroll
            for (int k = 0; k < kPix; k++) {
                float v = rnd<T>(acc[o][k]) + bias[o];
                if (fabsf(v) > p.clamp) {
                    v = v < 0.f ? -p.clamp : p.clamp;
                    code[k] |= 1u << o;
                }
                out[k] = v;
            }
            store_run(ys + o * hw, vec, nv, out);
        }
        if (p.mask) {
            unsigned char* m = p.mask + tl.np * hw + pix;
            if (vec) {
                *reinterpret_cast<uint2*>(m) = make_uint2(code[0] | code[1] << 8 | code[2] << 16 | code[3] << 24,
                                                          code[4] | code[5] << 8 | code[6] << 16 | code[7] << 24);
            } else {
#pragma unroll
                for (int k = 0; k < kPix; k++)
                    if (k < nv) m[k] = (unsigned char)code[k];
            }
        }
    }
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <class TX, class T>
__global__ void __launch_bounds__(kThreads, 2) sres_torgb_backward_kernel(const TorgbParams p)
{
    extern __shared__ __align__(16) float smem_b[];
    const Tile<T> tl(p, smem_b, true);
    const int64_t hw = (int64_t)p.ah.out * p.aw.out;
    const bool vec = p.vec != 0;
    const float* wf = smem_b + tl.L.wf;
    const float* af = smem_b + tl.L.af;
    float* red = smem_b + tl.L.red;                                      // [kWarps][4 cin + 3]
    const int nq = 4 * p.cin + kCout;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const TX* __restrict__ xs = reinterpret_cast<const TX*>(p.x) + tl.np * p.c * hw;
    TX* dxs = reinterpret_cast<TX*>(p.dx) + tl.np * p.c * hw;
    const T* dys = reinterpret_cast<const T*>(p.dy) + tl.np * kCout * hw;
    const unsigned char* ms = p.mask + tl.np * hw;

    // one run per thread: the tile has at most kThreads runs (host), so every thread takes part in each warp sum once
    const int q0 = threadIdx.x * kPix;
    const int nv = max(0, min(kPix, tl.npix - q0));
    const int64_t pix = tl.pix0 + q0;
    float g[kCout][kPix];
    {
        unsigned m[kPix];
        if (nv > 0) {
#pragma unroll
            for (int k = 0; k < kPix; k++) m[k] = k < nv ? ms[pix + k] : 0u;
#pragma unroll
            for (int o = 0; o < kCout; o++) load_run(dys + o * hw + pix, vec, nv, g[o]);
        } else {
#pragma unroll
            for (int k = 0; k < kPix; k++) m[k] = 0u;
#pragma unroll
            for (int o = 0; o < kCout; o++)
#pragma unroll
                for (int k = 0; k < kPix; k++) g[o][k] = 0.f;
        }
#pragma unroll
        for (int o = 0; o < kCout; o++)
#pragma unroll
            for (int k = 0; k < kPix; k++)
                if ((m[k] >> o) & 1u) g[o][k] = 0.f;
    }
#pragma unroll
    for (int o = 0; o < kCout; o++) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kPix; k++) s += g[o][k];
        s = warp_sum(s);
        if (lane == 0) red[warp * nq + 4 * p.cin + o] = s;
    }
    int roff[kPix], toff[kPix];
    if (p.cc > 0) run_offsets(p, nv > 0 ? q0 : 0, roff, toff);

    for (int ch = 0; ch < p.cin; ch++) {
        const bool from_x = ch < p.c;
        float z[kPix];
        if (from_x) {
            float v[kPix];
            if (nv > 0) load_run(xs + ch * hw + pix, vec, nv, v);
            else
#pragma unroll
                for (int k = 0; k < kPix; k++) v[k] = 0.f;
#pragma unroll
            for (int k = 0; k < kPix; k++) z[k] = rnd<T>(v[k]);
        } else {
            tl.cond_run(p, ch - p.c, roff, toff, nv, z);
        }
        const float a = af[ch], w0 = wf[ch], w1 = wf[p.cin + ch], w2 = wf[2 * p.cin + ch];
        float sa = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f, dxo[kPix];
#pragma unroll
        for (int k = 0; k < kPix; k++) {
            const float az = rnd<T>(z[k] * a);
            const float dxp = rnd<T>(fmaf(w2, g[2][k], fmaf(w1, g[1][k], w0 * g[0][k])));
            sa = fmaf(dxp, z[k], sa);
            s0 = fmaf(g[0][k], az, s0);
            s1 = fmaf(g[1][k], az, s1);
            s2 = fmaf(g[2][k], az, s2);
            dxo[k] = rnd<T>(dxp * a);
        }
        if (from_x && p.dx && nv > 0) store_run(dxs + ch * hw + pix, vec, nv, dxo);
        sa = warp_sum(sa);
        s0 = warp_sum(s0);
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        if (lane == 0) {
            float* r = red + warp * nq;
            r[ch] = sa;
            r[p.cin + ch] = s0;
            r[2 * p.cin + ch] = s1;
            r[3 * p.cin + ch] = s2;
        }
    }
    __syncthreads();
    float* out = p.part + (int64_t)blockIdx.x * nq;
    for (int q = threadIdx.x; q < nq; q += kThreads) {
        float s = 0.f;
        for (int k = 0; k < kWarps; k++) s += red[k * nq + q];
        out[q] = s;
    }
}

// per sample: the sum over its row tiles, in tile order. da goes to its output, the Gram rows and dy' sums to sums
__global__ void __launch_bounds__(256) sres_torgb_fold_tiles_kernel(const float* __restrict__ part, int64_t np, int row_tiles, int cin,
                                                                    float* __restrict__ da, float* __restrict__ sums)
{
    const int nq = 4 * cin + kCout;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= np * nq) return;
    const int64_t s = idx / nq;
    const int q = (int)(idx % nq);
    const float* src = part + s * row_tiles * nq + q;
    float acc = 0.f;
    for (int k = 0; k < row_tiles; k++) acc += src[(int64_t)k * nq];
    if (q < cin) da[s * cin + q] = acc;
    else sums[s * (nq - cin) + (q - cin)] = acc;
}

// dw [3][cin] and db [3] in the layer dtype: the per-sample sums added in sample order
template <class T>
__global__ void __launch_bounds__(256) sres_torgb_fold_samples_kernel(const float* __restrict__ sums, int64_t np, int cin,
                                                                      T* __restrict__ dw, T* __restrict__ db)
{
    const int nq = 3 * cin + kCout;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    float acc = 0.f;
    for (int64_t s = 0; s < np; s++) acc += sums[s * nq + q];
    if (q < 3 * cin) {
        if (dw) dw[q] = from_acc<T>(acc);
    } else if (db) {
        db[q - 3 * cin] = from_acc<T>(acc);
    }
}

struct Torgb {
    int64_t np, hw;
    int n, t, c, cin, cc, window;
    int rows, row_tiles;
    int64_t smem_fwd, smem_bwd;
    sres::Axis ah, aw;
};

bool torgb_plan(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr, const int* plan_h, const int* plan_w,
                int cout, Torgb& T)
{
    if (dtype != LVG_F16 && dtype != LVG_F32) return false;
    if (cout != kCout || n < 1 || t < 1 || c < 0 || c_lr < 1 || window < 1 || !plan_h || !plan_w) return false;
    if ((int64_t)c + (int64_t)c_lr * window > kMaxCin || (int64_t)t + window - 1 > t_lr) return false;
    if (!sres::read_axis(plan_h, h_lr, T.ah) || !sres::read_axis(plan_w, w_lr, T.aw)) return false;
    // the conditioning must be one lvg_sres_cond takes (the same plan checks, shared-memory tap tables)
    if (lvg_sres_cond_workspace(n, t, 0, c_lr, window, t_lr, h_lr, w_lr, dtype, plan_h, plan_w) < 0) return false;
    T.n = n; T.t = t; T.c = c; T.cc = c_lr * window; T.cin = c + T.cc; T.window = window;
    T.np = (int64_t)n * t;
    T.hw = (int64_t)T.ah.out * T.aw.out;
    if ((T.np * std::max(T.cin, kCout) * T.hw) >> 40 || T.np > (1 << 24)) return false;
    // rows per CTA: at most kTilePix pixels (one run per thread), fewer while the tile's shared memory does not fit
    for (T.rows = std::min<int>(T.ah.out, std::max(1, kTilePix / T.aw.out)); T.rows >= 1; T.rows--) {
        T.smem_bwd = tile_smem(T.cc, T.rows, w_lr, T.ah.nt, T.aw.out, T.aw.nt, T.cin, true).total;
        if (T.smem_bwd <= kMaxSmem) break;
    }
    if (T.rows < 1 || (int64_t)T.rows * T.aw.out > kTilePix) return false;
    T.smem_fwd = tile_smem(T.cc, T.rows, w_lr, T.ah.nt, T.aw.out, T.aw.nt, T.cin, false).total;
    T.row_tiles = (T.ah.out + T.rows - 1) / T.rows;
    if (T.np * T.row_tiles >= (1ll << 31)) return false;
    return true;
}

int64_t round256(int64_t v) { return (v + 255) / 256 * 256; }

struct TorgbRooms {
    int64_t part, sums;
    int64_t total() const { return part + sums; }
};
TorgbRooms torgb_rooms(const Torgb& T)
{
    const int64_t nq = 4 * T.cin + kCout;
    return {round256(T.np * T.row_tiles * nq * 4), round256(T.np * (nq - T.cin) * 4)};
}

TorgbParams torgb_params(const Torgb& T, const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                         const int64_t* st, float gain_h, float gain_w)
{
    TorgbParams p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.lr = lr; p.w = w; p.a = a;
    p.s_n = st[0]; p.s_c = st[1]; p.s_t = st[2]; p.s_h = st[3]; p.s_w = st[4];
    p.t = T.t; p.c = T.c; p.cin = T.cin; p.cc = T.cc; p.window = T.window;
    p.rows = T.rows; p.row_tiles = T.row_tiles;
    p.ah = T.ah; p.aw = T.aw;
    p.ah.f = f_h; p.ah.gain = gain_h;
    p.aw.f = f_w; p.aw.gain = gain_w;
    return p;
}

template <class K>
int launch_tile(K kern, const Torgb& T, int64_t smem, const TorgbParams& p, cudaStream_t s)
{
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)(T.np * T.row_tiles), kThreads, (size_t)smem, s>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

bool aligned_to(const void* p, int64_t bytes) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_sres_torgb_workspace(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                            const int* plan_h, const int* plan_w, int cout)
{
    Torgb T;
    if (!torgb_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, T)) return -1;
    return torgb_rooms(T).total();
}

extern "C" int lvg_sres_torgb_fprop(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                                    const void* b, void* y, unsigned char* mask, int x_dtype, int dtype, int n, int t, int c, int c_lr,
                                    int window, int t_lr, int h_lr, int w_lr, const int64_t* lr_strides, const int* plan_h,
                                    const int* plan_w, float gain_h, float gain_w, int cout, float clamp, void* stream)
{
    Torgb T;
    if (!torgb_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, T)) {
        set_error("sres_torgb_fprop: shape or plan outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x_dtype == LVG_F32 || x_dtype == LVG_F16, "sres_torgb_fprop: x_prev is fp32 or fp16");
    LVG_REQUIRE(lr && lr_strides && w && a && b && y && (c == 0 || x),
                "sres_torgb_fprop: lr, lr_strides, w, a, b, y (and x when c > 0) must not be NULL");
    LVG_REQUIRE((T.ah.ntaps == 0 || f_h) && (T.aw.ntaps == 0 || f_w), "sres_torgb_fprop: a filtered axis needs its filter");
    LVG_REQUIRE(!(clamp < 0.f), "sres_torgb_fprop: clamp must not be negative");
    const int xs = x_dtype == LVG_F32 ? 4 : 2, es = dtype == LVG_F32 ? 4 : 2;
    LVG_REQUIRE(aligned_to(x, xs) && aligned_to(y, es), "sres_torgb_fprop: x or y is not aligned to its element");
    TorgbParams p = torgb_params(T, x, lr, f_h, f_w, w, a, lr_strides, gain_h, gain_w);
    p.b = b; p.y = y; p.mask = mask; p.clamp = clamp;
    p.vec = T.aw.out % kPix == 0 && aligned16(x) && aligned16(y) && aligned_to(mask, 8);
    cudaStream_t s = (cudaStream_t)stream;
    void (*const kerns[2][2])(const TorgbParams) = {
        {sres_torgb_fprop_kernel<__half, __half>, sres_torgb_fprop_kernel<__half, float>},
        {sres_torgb_fprop_kernel<float, __half>, sres_torgb_fprop_kernel<float, float>}};
    return launch_tile(kerns[x_dtype == LVG_F32][dtype == LVG_F32], T, T.smem_fwd, p, s);
}

extern "C" int lvg_sres_torgb_backward(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                                       const unsigned char* mask, const void* dy, void* dx, void* dw, float* da, void* db, int x_dtype,
                                       int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                       const int64_t* lr_strides, const int* plan_h, const int* plan_w, float gain_h, float gain_w,
                                       int cout, void* workspace, int64_t workspace_bytes, void* stream)
{
    Torgb T;
    if (!torgb_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, T)) {
        set_error("sres_torgb_backward: shape or plan outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x_dtype == LVG_F32 || x_dtype == LVG_F16, "sres_torgb_backward: x_prev is fp32 or fp16");
    LVG_REQUIRE(lr && lr_strides && w && a && mask && dy && da && (c == 0 || x),
                "sres_torgb_backward: lr, lr_strides, w, a, mask, dy, da (and x when c > 0) must not be NULL");
    LVG_REQUIRE((T.ah.ntaps == 0 || f_h) && (T.aw.ntaps == 0 || f_w), "sres_torgb_backward: a filtered axis needs its filter");
    const int xs = x_dtype == LVG_F32 ? 4 : 2, es = dtype == LVG_F32 ? 4 : 2;
    LVG_REQUIRE(aligned_to(x, xs) && aligned_to(dx, xs) && aligned_to(dy, es), "sres_torgb_backward: x, dx or dy is not aligned to its element");
    const TorgbRooms r = torgb_rooms(T);
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.total(), "sres_torgb_backward: workspace too small or misaligned");
    TorgbParams p = torgb_params(T, x, lr, f_h, f_w, w, a, lr_strides, gain_h, gain_w);
    p.mask = const_cast<unsigned char*>(mask); p.dy = dy; p.dx = dx;
    p.part = reinterpret_cast<float*>(workspace);
    float* sums = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + r.part);
    p.vec = T.aw.out % kPix == 0 && aligned16(x) && aligned16(dx) && aligned16(dy) && aligned_to(mask, 8);
    cudaStream_t s = (cudaStream_t)stream;
    void (*const kerns[2][2])(const TorgbParams) = {
        {sres_torgb_backward_kernel<__half, __half>, sres_torgb_backward_kernel<__half, float>},
        {sres_torgb_backward_kernel<float, __half>, sres_torgb_backward_kernel<float, float>}};
    int rc = launch_tile(kerns[x_dtype == LVG_F32][dtype == LVG_F32], T, T.smem_bwd, p, s);
    if (rc) return rc;
    const int64_t nq = 4 * T.cin + kCout;
    sres_torgb_fold_tiles_kernel<<<(unsigned)((T.np * nq + 255) / 256), 256, 0, s>>>(p.part, T.np, T.row_tiles, T.cin, da, sums);
    LVG_LAUNCH_CHECK();
    const int nq2 = 3 * T.cin + kCout;
    if (dtype == LVG_F32)
        sres_torgb_fold_samples_kernel<float><<<(nq2 + 255) / 256, 256, 0, s>>>(sums, T.np, T.cin, (float*)dw, (float*)db);
    else
        sres_torgb_fold_samples_kernel<__half><<<(nq2 + 255) / 256, 256, 0, s>>>(sums, T.np, T.cin, (__half*)dw, (__half*)db);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}
