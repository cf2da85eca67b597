// Register-blocked separable polyphase FIR passes over shared-memory tiles.
//
// Building blocks of the single-launch separable upfirdn2d kernel
// (upfirdn2d_tiled.cu). Every pass reads a tile from shared memory,
// keeps the (compile-time sized) filter in registers and lets each thread
// produce a short run of outputs from one contiguous window of inputs, so a
// shared-memory load feeds ~4-5 FMAs instead of 1 (LDS issue rate is 1/4 of the
// FMA rate, so this is what keeps the FMA pipe, not the LSU, busy).
//
// Up-sampling passes work on the phase-aligned up-sampled axis: position
// a = UP*q + r (q = "group", r = phase) is
//     out[a] = sum_k g[(UP - r) % UP + k*UP] * in[q + (r > 0) + k],  k < F/UP
// which is zero-insertion + FIR with the zero taps removed (F % UP == 0).
// Down-sampling passes are plain strided correlations
//     out[o] = sum_t g[t] * in[o*DOWN + t],  t < F.
// g is the filter already oriented for correlation (mirrored unless flip).
//
// Lane mapping: passes along x give each warp W rows x (32/W) column groups
// where W is the per-thread advance in words, so with an odd row pitch the 32
// lanes of a load hit 32 distinct banks; passes along y map lanes to
// consecutive columns (stride 1).

#pragma once
#include "common.cuh"

namespace lvg {
namespace fir {

constexpr int kWarp = 32;

// n / d for small non-negative n without the integer-division sequence
struct FastDiv {
    unsigned magic;   // ceil(2^32 / d) = floor((2^32 - 1) / d) + 1 for d > 1 (32-bit division only); exact for n * d < 2^32
    int d;
    __host__ __device__ explicit FastDiv(int d_ = 1) : magic(d_ > 1 ? 0xFFFFFFFFu / (unsigned)d_ + 1u : 0u), d(d_) {}
    __device__ __forceinline__ int div(int n) const { return d > 1 ? (int)__umulhi((unsigned)n, magic) : n; }
};



// A y pass hands every result to an "emitter". Plain callables get emit(plane, row, col, value). Emitters made with
// make_emitter(begin, put) first get begin(plane, col) -> context ONCE per thread item (e.g. the column's base pointer)
// and then put(context, row, value) per result, which keeps 64-bit address arithmetic out of the per-result path.
template <class Begin, class Put> struct ItemEmitter { Begin begin; Put put; };
template <class Begin, class Put> __device__ __forceinline__ ItemEmitter<Begin, Put> make_emitter(Begin b, Put p) { return ItemEmitter<Begin, Put>{b, p}; }

template <class E> struct EmitCtx {
    int pl, col;
    __device__ __forceinline__ EmitCtx(E&, int pl_, int col_) : pl(pl_), col(col_) {}
    __device__ __forceinline__ void put(E& e, int row, float v) const { e(pl, row, col, v); }
};
template <class Begin, class Put> struct EmitCtx<ItemEmitter<Begin, Put>> {
    decltype(((Begin*)nullptr)->operator()(0, 0)) ctx;
    __device__ __forceinline__ EmitCtx(ItemEmitter<Begin, Put>& e, int pl, int col) : ctx(e.begin(pl, col)) {}
    __device__ __forceinline__ void put(ItemEmitter<Begin, Put>& e, int row, float v) const { e.put(ctx, row, v); }
};

// ---------------------------------------------------------------------------
// down-sampling along x.  in: [rows][pin] read from column offset `xoff`;
// out[r][o] = sum_t g[t] * in[r][xoff + o*DOWN + t], o < outs (rounded up to R).
template <int DOWN, int F, int R, int NTHREADS>
__device__ __forceinline__ void down_x(const float* __restrict__ in, int pin, int xoff, float* __restrict__ out, int pout,
                                       int rows, int outs, const float* __restrict__ s_taps)
{
    constexpr int ADV = R * DOWN;                       // per-thread input advance in words
    constexpr int RW = ADV >= kWarp ? kWarp : ADV;      // rows per warp
    constexpr int GW = kWarp / RW;
    constexpr int NIN = (R - 1) * DOWN + F;
    float g[F];
#pragma unroll
    for (int i = 0; i < F; i++) g[i] = s_taps[i];
    const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
    const int gthreads = (outs + R - 1) / R;
    const int n_rt = (rows + RW - 1) / RW, n_gt = (gthreads + GW - 1) / GW;
    const FastDiv by_gt(n_gt);
    for (int wi = warp; wi < n_rt * n_gt; wi += NTHREADS / kWarp) {
        const int rt = by_gt.div(wi), gt = wi - rt * n_gt;
        const int r = rt * RW + lane % RW;
        const int tg = gt * GW + lane / RW;
        if (r < rows && tg < gthreads) {
            const float* src = in + r * pin + xoff + tg * ADV;
            float v[NIN];
#pragma unroll
            for (int i = 0; i < NIN; i++) v[i] = src[i];
            float* dst = out + r * pout + tg * R;
#pragma unroll
            for (int j = 0; j < R; j++) {
                float acc = 0.f;
#pragma unroll
                for (int t = 0; t < F; t++) acc = fmaf(g[t], v[j * DOWN + t], acc);
                dst[j] = acc;
            }
        }
    }
}

// ---------------------------------------------------------------------------
// down-sampling along y.  in: [nplanes][plane_rows][pin] read from row offset `yoff` of each plane;
// value(plane, o, col) = sum_t g[t] * in[plane][yoff + o*DOWN + t][col] for o < outs, handed to `emit`.
template <int DOWN, int F, int R, int NTHREADS, class Emit>
__device__ __forceinline__ void down_y(const float* __restrict__ in, int pin, int yoff, int cols, int outs,
                                       const float* __restrict__ s_taps, Emit emit, int nplanes = 1, int plane_rows = 0)
{
    constexpr int NIN = (R - 1) * DOWN + F;
    float g[F];
#pragma unroll
    for (int i = 0; i < F; i++) g[i] = s_taps[i];
    const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
    const int gthreads = (outs + R - 1) / R;
    const int vcols = nplanes * cols;
    const int n_cc = (vcols + kWarp - 1) / kWarp;
    const FastDiv by_cols(cols), by_cc(n_cc);
    for (int wi = warp; wi < gthreads * n_cc; wi += NTHREADS / kWarp) {
        const int tg = by_cc.div(wi), cc = wi - tg * n_cc;
        const int vc = cc * kWarp + lane;
        if (vc < vcols) {
            const int pl = nplanes > 1 ? by_cols.div(vc) : 0;
            const int col = vc - pl * cols;
            const float* src = in + (pl * plane_rows + yoff + tg * R * DOWN) * pin + col;
            float v[NIN];
#pragma unroll
            for (int i = 0; i < NIN; i++) v[i] = src[i * pin];
#pragma unroll
            for (int j = 0; j < R; j++) {
                float acc = 0.f;
#pragma unroll
                for (int t = 0; t < F; t++) acc = fmaf(g[t], v[j * DOWN + t], acc);
                if (tg * R + j < outs) EmitCtx<Emit>(emit, pl, col).put(emit, tg * R + j, acc);
            }
        }
    }
}

// ===========================================================================================
// Paired variants: every thread produces TWO outputs per coefficient load, as two scalar FMAs
// (sm_90 has no packed f32x2 FMA), which halves the shared-memory reads of the inner loops.
// The two outputs of a pair lie along the axis that is NOT being filtered: rows r and r + RW of
// the same warp item (two conflict-free 32-bit loads). The paired y passes of upfirdn2d_tiled.cu
// pair columns L and L + 32 of a 64-column span instead. Coefficients are held as (g, g) pairs.

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <int UP, int F, int R, int NTHREADS>
__device__ __forceinline__ void up_x2(const float* __restrict__ in, int pin, float* __restrict__ out, int pout,
                                      int rows, int groups, const float* __restrict__ s_taps)
{
    static_assert(F % UP == 0, "filter length must be a multiple of the up-sampling factor");
    constexpr int K = F / UP;
    constexpr int RW = R;
    constexpr int GW = kWarp / RW;
    float2 g[F];
#pragma unroll
    for (int i = 0; i < F; i++) g[i] = make_float2(s_taps[i], s_taps[i]);
    const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
    const int gthreads = (groups + R - 1) / R;
    const int n_rt = (rows + 2 * RW - 1) / (2 * RW), n_gt = (gthreads + GW - 1) / GW;
    const FastDiv by_gt(n_gt);
    for (int wi = warp; wi < n_rt * n_gt; wi += NTHREADS / kWarp) {
        const int rt = by_gt.div(wi), gt = wi - rt * n_gt;
        const int ra = rt * 2 * RW + lane % RW;
        const int tg = gt * GW + lane / RW;
        if (ra < rows && tg < gthreads) {
            const bool has_b = ra + RW < rows;
            const float* sa = in + ra * pin + tg * R;
            const float* sb = has_b ? sa + RW * pin : sa;
            float2 v[K + R];
#pragma unroll
            for (int i = 0; i < K + R; i++) v[i] = make_float2(sa[i], sb[i]);
            float* da = out + ra * pout + tg * R * UP;
            float* db = da + RW * pout;
#pragma unroll
            for (int j = 0; j < R; j++) {
#pragma unroll
                for (int ph = 0; ph < UP; ph++) {
                    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                    for (int k = 0; k < K; k++)
                        acc = ffma2(g[(UP - ph) % UP + k * UP], v[j + (ph > 0 ? 1 : 0) + k], acc);
                    da[j * UP + ph] = acc.x;
                    if (has_b) db[j * UP + ph] = acc.y;
                }
            }
        }
    }
}

template <int DOWN, int F, int R, int NTHREADS>
__device__ __forceinline__ void down_x2(const float* __restrict__ in, int pin, int xoff, float* __restrict__ out, int pout,
                                        int rows, int outs, const float* __restrict__ s_taps)
{
    constexpr int ADV = R * DOWN;
    constexpr int RW = ADV >= kWarp ? kWarp : ADV;
    constexpr int GW = kWarp / RW;
    constexpr int NIN = (R - 1) * DOWN + F;
    float2 g[F];
#pragma unroll
    for (int i = 0; i < F; i++) g[i] = make_float2(s_taps[i], s_taps[i]);
    const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
    const int gthreads = (outs + R - 1) / R;
    const int n_rt = (rows + 2 * RW - 1) / (2 * RW), n_gt = (gthreads + GW - 1) / GW;
    const FastDiv by_gt(n_gt);
    for (int wi = warp; wi < n_rt * n_gt; wi += NTHREADS / kWarp) {
        const int rt = by_gt.div(wi), gt = wi - rt * n_gt;
        const int ra = rt * 2 * RW + lane % RW;
        const int tg = gt * GW + lane / RW;
        if (ra < rows && tg < gthreads) {
            const bool has_b = ra + RW < rows;
            const float* sa = in + ra * pin + xoff + tg * ADV;
            const float* sb = has_b ? sa + RW * pin : sa;
            float2 v[NIN];
#pragma unroll
            for (int i = 0; i < NIN; i++) v[i] = make_float2(sa[i], sb[i]);
            float* da = out + ra * pout + tg * R;
            float* db = da + RW * pout;
#pragma unroll
            for (int j = 0; j < R; j++) {
                float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                for (int t = 0; t < F; t++) acc = ffma2(g[t], v[j * DOWN + t], acc);
                da[j] = acc.x;
                if (has_b) db[j] = acc.y;
            }
        }
    }
}

__host__ __device__ constexpr int even_pitch(int w) { return (w + 1) & ~1; }

__host__ __device__ constexpr int odd_pitch(int w) { return w | 1; }
__host__ __device__ constexpr int round_up(int a, int b) { return (a + b - 1) / b * b; }

}  // namespace fir
}  // namespace lvg
