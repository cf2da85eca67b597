// Tail of the low-res discriminator's residual block (DiscriminatorBlock.forward after conv_1's convolution,
// discriminator_lres.py:321-333 with Conv3dLayer.forward :169-179 and Downsample3d.forward :197-213) as one op:
//
//   z = scale * (bias_act(P y, b, act, gain, clamp) + s)          scale = sqrt(1/2) with MERGE, else 1 and no s
//
// y [n][c][t][h][w] is the convolution output, s the skip tensor at the output resolution. P is, per axis, a copy or
// Downsample3d's filter   out[m] = sum_j f[3 - j] * in[2 m - 1 + j]   (zero outside, even extents), fir3d.cu's operator
// with (filt, step, off) = (1, 2, -1), on T (TDOWN) and / or on H and W (SDOWN).
//
// The map is piecewise linear. With G the activation slopes (gain, gain * alpha, 0 where clamped) two kernels close its
// gradients of every order:
//   forward   write: z and 2-bit codes per output (bit 0 not positive, bit 1 clamped, evaluated on the value bias_act
//             stores, as bias_act evaluates them); none: z only. In both, bias_act's output is rounded to the storage type
//             before s is added, as the composition stores it; the sum and the scale then round once;
//             read: scale * (G (P u + beta) + sigma) with G from codes.
//   adjoint   dv = scale * G dz, dy = P^T dv, ds = scale * dz (optional), db[c] = sum of dv.
//
// Both are fir3d.cu's walk: one CTA owns an (n, c) plane and an 8 x 32 tile of output rows x columns and walks the frames
// once, so each input frame is read once; H and W filter through shared memory, T over a register window. The forward
// applies bias, activation and the merge where fir3d stores; the adjoint applies scale * G while it stages dz. Every
// element of dz belongs to exactly one CTA (the one whose tile of dy holds its first full-rate sample), which writes its ds
// and adds its dv to one partial sum per CTA; a second kernel folds the partials per channel in a fixed order. No atomics,
// and the partition into partials depends on the shape only: results are bitwise reproducible.
//
// Codes: one byte per 4 consecutive outputs along W (element k of the group in bits 2k, 2k + 1), rows padded to
// ceil(w_out / 4) bytes, rows in the order of z.
#include "common.cuh"
#include "fir3d_axis.cuh"

namespace lvg {
namespace {

using namespace fir3d_axis;

constexpr float kSqrtHalf = 0.70710678118654752440f;
// the adjoint stages at most kTH x kTW elements of dz per frame (8 x 32 unfiltered, 6 x 18 with both axes filtered)
constexpr int kAdjLoads = 1;

struct TailArgs {
    const float* f;
    const float* b;
    int c;
    Axis at, ah, aw;
    float alpha, gain, clamp;       // forward decision (write / none)
    float slope_pos, slope_neg;     // G where not clamped (read, adjoint)
    float scale;
    int code_row;                   // bytes per row of codes
};

__device__ __forceinline__ float slope_of(unsigned code, const TailArgs& a)
{
    return (code & 2u) ? 0.f : (code & 1u) ? a.slope_neg : a.slope_pos;
}

// codes of a value bias_act stored (bias_act.cu's decision on the rounded output)
template <class T>
__device__ __forceinline__ unsigned code_of(float o, const TailArgs& a)
{
    const float ys = to_acc(from_acc<T>(o));
    const float inv_gain = a.gain != 0.f ? 1.f / a.gain : 0.f;
    unsigned code = (inv_gain > 0.f ? !(ys > 0.f) : !(ys * inv_gain > 0.f)) ? 1u : 0u;
    if (a.clamp >= 0.f && !(fabsf(ys) < a.clamp)) code |= 2u;
    return code;
}

template <class T, int MODE>
__global__ void __launch_bounds__(kThreads) dblock_tail_fwd_kernel(const T* __restrict__ y, const T* __restrict__ s, T* __restrict__ z,
                                                                  uint8_t* __restrict__ codes, TailArgs a)
{
    __shared__ float sa[kRows][kCols + 1];
    __shared__ float sb[kTH][kCols + 1];
    float g[4];
#pragma unroll
    for (int j = 0; j < 4; j++) g[j] = a.f ? a.f[3 - j] : 0.f;      // no taps where no axis is filtered

    const Axis at = a.at, ah = a.ah, aw = a.aw;
    const int tin = at.n_in, tout = at.n_out, hin = ah.n_in, hout = ah.n_out, win_ = aw.n_in, wout = aw.n_out;
    const int nc = blockIdx.x, ci = nc % a.c;
    const int tiles_w = (wout + kTW - 1) / kTW;
    const int h0 = (blockIdx.y / tiles_w) * kTH, w0 = (blockIdx.y % tiles_w) * kTW;
    const int h1 = min(h0 + kTH, hout), w1 = min(w0 + kTW, wout);
    const int r_lo = ax_base<false>(ah, h0), c_lo = ax_base<false>(aw, w0);
    const int nrows = ax_base<false>(ah, h1 - 1) + ax_ntaps<false>(ah) - r_lo;
    const int ncols = ax_base<false>(aw, w1 - 1) + ax_ntaps<false>(aw) - c_lo;
    const int nth = ax_ntaps<false>(ah), ntw = ax_ntaps<false>(aw), ntt = ax_ntaps<false>(at);

    const int tid = threadIdx.x, my_r = tid / kTW, my_q = tid % kTW;
    const bool mine = h0 + my_r < h1 && w0 + my_q < w1;
    const int mw = w0 + my_q;
    const int bw = ax_base<false>(aw, mw) - c_lo;
    const float bias = a.b ? a.b[ci] : 0.f;
    const int64_t plane_in = (int64_t)hin * win_;

    float win[4] = {0.f, 0.f, 0.f, 0.f};     // filtered frames base_t .. base_t + 3 at this thread's output pixel
    int loaded = ax_base<false>(at, 0) - 1;
    for (int mt = 0; mt < tout; mt++) {
        const int bt = ax_base<false>(at, mt);
        while (loaded < bt + ntt - 1) {       // block-uniform
            ++loaded;
            float v = 0.f;
            if (loaded >= 0 && loaded < tin) {
                const T* xf = y + ((int64_t)nc * tin + loaded) * plane_in;
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
                    float acc = 0.f;
                    if (m < h1) {
                        const int bb = ax_base<false>(ah, m) - r_lo;
#pragma unroll
                        for (int r = 0; r < 4; r++)
                            if (r < nth) acc = fmaf(ax_tap<false>(ah, g, m, r), sa[bb + r][cc], acc);
                    }
                    sb[rr][cc] = acc;
                }
                __syncthreads();
                if (mine) {
#pragma unroll
                    for (int r = 0; r < 4; r++)
                        if (r < ntw) v = fmaf(ax_tap<false>(aw, g, mw, r), sb[my_r][bw + r], v);
                }
            }
#pragma unroll
            for (int r = 0; r < 3; r++) win[r] = win[r + 1];
            win[3] = v;
        }
        // the window ends at frame `loaded` = bt + ntt - 1: tap r of this output sits in win[4 - ntt + r]
        unsigned code = 0;
        if (mine) {
            float acc = 0.f;
#pragma unroll
            for (int r = 0; r < 4; r++)
                if (r >= 4 - ntt) acc = fmaf(at.filt ? g[r] : 1.f, win[r], acc);
            const int64_t row = ((int64_t)nc * tout + mt) * hout + (h0 + my_r);
            const int64_t e = row * wout + mw;
            const float x = __fadd_rn(acc, bias);
            float o;
            if (MODE == LVG_DBLOCK_TAIL_READ) {
                code = (codes[row * a.code_row + (mw >> 2)] >> (2 * (mw & 3))) & 3u;
                o = __fmul_rn(x, slope_of(code, a));
            } else {
                o = __fmul_rn(x > 0.f ? x : __fmul_rn(x, a.alpha), a.gain);
                if (a.clamp >= 0.f) o = (o > -a.clamp && o < a.clamp) ? o : (o >= 0.f ? a.clamp : -a.clamp);
                o = to_acc(from_acc<T>(o));           // bias_act stores its output in T before the merge reads it
                if (MODE == LVG_DBLOCK_TAIL_WRITE) code = code_of<T>(o, a);
            }
            if (s) o = __fadd_rn(o, to_acc(s[e]));
            z[e] = from_acc<T>(__fmul_rn(o, a.scale));
        }
        if (MODE == LVG_DBLOCK_TAIL_WRITE) {  // a warp is one row of the tile: 4 neighbouring lanes share a byte
            unsigned byte = code << (2 * (tid & 3));
            byte |= __shfl_xor_sync(0xffffffffu, byte, 1);
            byte |= __shfl_xor_sync(0xffffffffu, byte, 2);
            if (mine && (tid & 3) == 0)
                codes[(((int64_t)nc * tout + mt) * hout + (h0 + my_r)) * a.code_row + (mw >> 2)] = (uint8_t)byte;
        }
    }
}

// range of P's output indices whose first full-rate sample lies in [m0, m1) (m0 a multiple of the tile, m1 even where the
// axis is filtered): the elements of dz a tile of dy owns
__device__ __forceinline__ void own_range(const Axis& a, int m0, int m1, int& lo, int& hi)
{
    lo = a.filt ? m0 >> 1 : m0;
    hi = a.filt ? m1 >> 1 : m1;
}

template <class T, bool DS>
__global__ void __launch_bounds__(kThreads) dblock_tail_adj_kernel(const T* __restrict__ dz, const uint8_t* __restrict__ codes,
                                                                  T* __restrict__ dy, T* __restrict__ ds, float* __restrict__ part,
                                                                  TailArgs a)
{
    __shared__ float sa[kRows][kCols + 1];
    __shared__ float sb[kTH][kCols + 1];
    __shared__ float swarp[kThreads / 32];
    float g[4];
#pragma unroll
    for (int j = 0; j < 4; j++) g[j] = a.f ? a.f[3 - j] : 0.f;      // no taps where no axis is filtered

    const Axis at = a.at, ah = a.ah, aw = a.aw;
    // extents as this kernel reads (dz) / writes (dy) them
    const int tin = at.n_out, tout = at.n_in, hin = ah.n_out, hout = ah.n_in, win_ = aw.n_out, wout = aw.n_in;
    const int nc = blockIdx.x;
    const int tiles_w = (wout + kTW - 1) / kTW;
    const int h0 = (blockIdx.y / tiles_w) * kTH, w0 = (blockIdx.y % tiles_w) * kTW;
    const int h1 = min(h0 + kTH, hout), w1 = min(w0 + kTW, wout);
    const int r_lo = ax_base<true>(ah, h0), c_lo = ax_base<true>(aw, w0);
    const int nrows = ax_base<true>(ah, h1 - 1) + ax_ntaps<true>(ah) - r_lo;
    const int ncols = ax_base<true>(aw, w1 - 1) + ax_ntaps<true>(aw) - c_lo;
    const int nth = ax_ntaps<true>(ah), ntw = ax_ntaps<true>(aw), ntt = ax_ntaps<true>(at);
    int or0, or1, oc0, oc1;
    own_range(ah, h0, h1, or0, or1);
    own_range(aw, w0, w1, oc0, oc1);

    const int tid = threadIdx.x, my_r = tid / kTW, my_q = tid % kTW;
    const bool mine = h0 + my_r < h1 && w0 + my_q < w1;
    const int mw = w0 + my_q;
    const int bw = ax_base<true>(aw, mw) - c_lo;
    float tw[2];
#pragma unroll
    for (int r = 0; r < 2; r++) tw[r] = r < ntw ? ax_tap<true>(aw, g, mw, r) : 0.f;

    const int64_t plane_in = (int64_t)hin * win_, plane_out = (int64_t)hout * wout;
    float sum = 0.f;                         // dv over the elements of dz this thread staged and the tile owns
    float win[2] = {0.f, 0.f};               // frames base_t, base_t + 1 of H^T W^T dv at this thread's pixel
    int loaded = ax_base<true>(at, 0) - 1;
    for (int mt = 0; mt < tout; mt++) {
        const int bt = ax_base<true>(at, mt);
        while (loaded < bt + ntt - 1) {       // block-uniform
            ++loaded;
            float v = 0.f;
            if (loaded >= 0 && loaded < tin) {
                const int64_t frame = (int64_t)nc * tin + loaded;
                const T* xf = dz + frame * plane_in;
                float ld[kAdjLoads];
#pragma unroll
                for (int k = 0; k < kAdjLoads; k++) {
                    const int idx = tid + k * kThreads;
                    const int rr = idx / ncols, cc = idx - rr * ncols, gr = r_lo + rr, gc = c_lo + cc;
                    ld[k] = 0.f;
                    if (rr < nrows && gr >= 0 && gr < hin && gc >= 0 && gc < win_) {
                        const float d = __fmul_rn(to_acc(xf[(int64_t)gr * win_ + gc]), a.scale);
                        const unsigned code = (codes[(frame * hin + gr) * a.code_row + (gc >> 2)] >> (2 * (gc & 3))) & 3u;
                        const float dv = __fmul_rn(d, slope_of(code, a));
                        ld[k] = dv;
                        if (gr >= or0 && gr < or1 && gc >= oc0 && gc < oc1) {
                            sum += dv;
                            if (DS) ds[frame * plane_in + (int64_t)gr * win_ + gc] = from_acc<T>(d);
                        }
                    }
                }
#pragma unroll
                for (int k = 0; k < kAdjLoads; k++) {
                    const int idx = tid + k * kThreads;
                    const int rr = idx / ncols;
                    if (rr < nrows) sa[rr][idx - rr * ncols] = ld[k];
                }
                __syncthreads();
                for (int idx = tid; idx < kTH * ncols; idx += kThreads) {
                    const int rr = idx / ncols, cc = idx - rr * ncols, m = h0 + rr;
                    float acc = 0.f;
                    if (m < h1) {
                        const int bb = ax_base<true>(ah, m) - r_lo;
#pragma unroll
                        for (int r = 0; r < 2; r++)
                            if (r < nth) acc = fmaf(ax_tap<true>(ah, g, m, r), sa[bb + r][cc], acc);
                    }
                    sb[rr][cc] = acc;
                }
                __syncthreads();
                if (mine) {
#pragma unroll
                    for (int r = 0; r < 2; r++)
                        if (r < ntw) v = fmaf(tw[r], sb[my_r][bw + r], v);
                }
            }
            win[0] = win[1];
            win[1] = v;
        }
        if (mine) {
            float acc = 0.f;
#pragma unroll
            for (int r = 0; r < 2; r++)
                if (r >= 2 - ntt) acc = fmaf(at.filt ? ax_tap<true>(at, g, mt, r) : 1.f, win[r], acc);
            dy[((int64_t)nc * tout + mt) * plane_out + (int64_t)(h0 + my_r) * wout + mw] = from_acc<T>(acc);
        }
    }

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((tid & 31) == 0) swarp[tid >> 5] = sum;
    __syncthreads();
    if (tid == 0) {
        float total = 0.f;
        for (int k = 0; k < kThreads / 32; k++) total += swarp[k];
        part[(int64_t)nc * gridDim.y + blockIdx.y] = total;
    }
}

// db[c] = sum over n and tiles of the CTAs' partial sums, in a fixed order
__global__ void __launch_bounds__(kThreads) dblock_tail_fold_kernel(const float* __restrict__ part, float* __restrict__ db, int n,
                                                                   int c, int tiles)
{
    const int ch = blockIdx.x * kThreads + threadIdx.x;
    if (ch >= c) return;
    float sum = 0.f;
    for (int i = 0; i < n; i++) {
        const float* q = part + ((int64_t)i * c + ch) * tiles;
        for (int k = 0; k < tiles; k++) sum += q[k];
    }
    db[ch] = sum;
}

struct Plan {
    Axis ax[3];
    int64_t tiles_fwd, tiles_adj;
    int code_row;
    int64_t code_bytes, ws_bytes;
};

// false when the shape is outside the op's envelope
bool make_plan(int n, int c, int t, int h, int w, int flags, Plan& pl)
{
    if (n < 1 || c < 1 || t < 1 || h < 1 || w < 1 || (flags & ~7) || (int64_t)n * c > 0x7fffffff) return false;
    const bool td = flags & LVG_DBLOCK_TAIL_TDOWN, sd = flags & LVG_DBLOCK_TAIL_SDOWN;
    const int in[3] = {t, h, w};
    const bool down[3] = {td, sd, sd};
    for (int i = 0; i < 3; i++) {
        if (down[i] && (in[i] & 1)) return false;
        pl.ax[i] = down[i] ? Axis{1, 2, -1, in[i], in[i] / 2} : Axis{0, 1, 0, in[i], in[i]};
    }
    auto tiles = [](int hh, int ww) { return (int64_t)((hh + kTH - 1) / kTH) * ((ww + kTW - 1) / kTW); };
    pl.tiles_fwd = tiles(pl.ax[1].n_out, pl.ax[2].n_out);
    pl.tiles_adj = tiles(h, w);
    if (pl.tiles_fwd > 65535 || pl.tiles_adj > 65535) return false;
    pl.code_row = (pl.ax[2].n_out + 3) / 4;
    pl.code_bytes = (int64_t)n * c * pl.ax[0].n_out * pl.ax[1].n_out * pl.code_row;
    pl.ws_bytes = ((int64_t)n * c * pl.tiles_adj * (int64_t)sizeof(float) + 15) & ~(int64_t)15;
    return true;
}

int check_call(const char* name, int dtype, int act)
{
    LVG_REQUIRE(dtype == LVG_F32 || dtype == LVG_F16, "%s: fp32 / fp16 only (got dtype %d)", name, dtype);
    if (act != LVG_ACT_LRELU && act != LVG_ACT_LINEAR) {
        set_error("%s: lrelu / linear only (got activation %d)", name, act);
        return LVG_UNSUPPORTED;
    }
    return LVG_OK;
}

TailArgs args_of(const Plan& pl, const float* f, const float* b, int c, int flags, int act, float alpha, float gain, float clamp)
{
    TailArgs a;
    memset(&a, 0, sizeof(a));
    a.f = f; a.b = b; a.c = c;
    a.at = pl.ax[0]; a.ah = pl.ax[1]; a.aw = pl.ax[2];
    a.alpha = act == LVG_ACT_LRELU ? alpha : 1.f;
    a.gain = gain; a.clamp = clamp;
    a.slope_pos = gain;
    a.slope_neg = gain * a.alpha;
    a.scale = (flags & LVG_DBLOCK_TAIL_MERGE) ? kSqrtHalf : 1.f;
    a.code_row = pl.code_row;
    return a;
}

template <class T>
int launch_fwd(const void* y, const void* s, void* z, uint8_t* codes, int mode, const TailArgs& a, dim3 grid, cudaStream_t st)
{
    const T *py = (const T*)y, *ps = (const T*)s;
    T* pz = (T*)z;
    if (mode == LVG_DBLOCK_TAIL_WRITE) dblock_tail_fwd_kernel<T, LVG_DBLOCK_TAIL_WRITE><<<grid, kThreads, 0, st>>>(py, ps, pz, codes, a);
    else if (mode == LVG_DBLOCK_TAIL_READ) dblock_tail_fwd_kernel<T, LVG_DBLOCK_TAIL_READ><<<grid, kThreads, 0, st>>>(py, ps, pz, codes, a);
    else dblock_tail_fwd_kernel<T, LVG_DBLOCK_TAIL_NONE><<<grid, kThreads, 0, st>>>(py, ps, pz, codes, a);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

template <class T>
int launch_adj(const void* dz, const uint8_t* codes, void* dy, void* ds, float* part, const TailArgs& a, dim3 grid, cudaStream_t st)
{
    if (ds) dblock_tail_adj_kernel<T, true><<<grid, kThreads, 0, st>>>((const T*)dz, codes, (T*)dy, (T*)ds, part, a);
    else dblock_tail_adj_kernel<T, false><<<grid, kThreads, 0, st>>>((const T*)dz, codes, (T*)dy, (T*)nullptr, part, a);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_dblock_tail_workspace(int n, int c, int t, int h, int w, int flags)
{
    Plan pl;
    return make_plan(n, c, t, h, w, flags, pl) ? pl.ws_bytes : LVG_UNSUPPORTED;
}

extern "C" int64_t lvg_dblock_tail_codes_bytes(int n, int c, int t, int h, int w, int flags)
{
    Plan pl;
    return make_plan(n, c, t, h, w, flags, pl) ? pl.code_bytes : LVG_UNSUPPORTED;
}

extern "C" int lvg_dblock_tail(const void* y, const void* s, const float* b, const float* f, void* z, uint8_t* codes, int mode,
                               int dtype, int n, int c, int t, int h, int w, int flags, int act, float alpha, float gain,
                               float clamp, void* stream)
{
    int rc = check_call("dblock_tail", dtype, act);
    if (rc) return rc;
    LVG_REQUIRE(y && z, "dblock_tail: y and z must not be NULL");
    LVG_REQUIRE(f || !(flags & (LVG_DBLOCK_TAIL_TDOWN | LVG_DBLOCK_TAIL_SDOWN)), "dblock_tail: f must not be NULL where an axis is filtered");
    LVG_REQUIRE(mode == LVG_DBLOCK_TAIL_NONE || mode == LVG_DBLOCK_TAIL_WRITE || mode == LVG_DBLOCK_TAIL_READ,
                "dblock_tail: mode must be 0 (none), 1 (write) or 2 (read)");
    LVG_REQUIRE((mode == LVG_DBLOCK_TAIL_NONE) == (codes == nullptr), "dblock_tail: codes are needed in write and read mode only");
    LVG_REQUIRE((flags & LVG_DBLOCK_TAIL_MERGE) || !s, "dblock_tail: s needs LVG_DBLOCK_TAIL_MERGE");
    Plan pl;
    if (!make_plan(n, c, t, h, w, flags, pl)) {
        set_error("dblock_tail: shape outside the envelope (n %d c %d t %d h %d w %d, flags %d)", n, c, t, h, w, flags);
        return LVG_UNSUPPORTED;
    }
    const TailArgs a = args_of(pl, f, b, c, flags, act, alpha, gain, clamp);
    const dim3 grid((unsigned)(n * c), (unsigned)pl.tiles_fwd);
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == LVG_F32 ? launch_fwd<float>(y, s, z, codes, mode, a, grid, st) : launch_fwd<__half>(y, s, z, codes, mode, a, grid, st);
}

extern "C" int lvg_dblock_tail_adjoint(const void* dz, const uint8_t* codes, const float* f, void* dy, void* ds, float* db,
                                       void* workspace, int64_t workspace_bytes, int dtype, int n, int c, int t, int h, int w,
                                       int flags, int act, float alpha, float gain, void* stream)
{
    int rc = check_call("dblock_tail_adjoint", dtype, act);
    if (rc) return rc;
    LVG_REQUIRE(dz && codes && dy && db && workspace, "dblock_tail_adjoint: dz, codes, dy, db and workspace must not be NULL");
    LVG_REQUIRE(f || !(flags & (LVG_DBLOCK_TAIL_TDOWN | LVG_DBLOCK_TAIL_SDOWN)), "dblock_tail_adjoint: f must not be NULL where an axis is filtered");
    Plan pl;
    if (!make_plan(n, c, t, h, w, flags, pl)) {
        set_error("dblock_tail_adjoint: shape outside the envelope (n %d c %d t %d h %d w %d, flags %d)", n, c, t, h, w, flags);
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(workspace_bytes >= pl.ws_bytes, "dblock_tail_adjoint: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                (long long)pl.ws_bytes);
    const TailArgs a = args_of(pl, f, nullptr, c, flags, act, alpha, gain, -1.f);
    const dim3 grid((unsigned)(n * c), (unsigned)pl.tiles_adj);
    cudaStream_t st = (cudaStream_t)stream;
    rc = dtype == LVG_F32 ? launch_adj<float>(dz, codes, dy, ds, (float*)workspace, a, grid, st)
                          : launch_adj<__half>(dz, codes, dy, ds, (float*)workspace, a, grid, st);
    if (rc) return rc;
    dblock_tail_fold_kernel<<<(unsigned)((c + kThreads - 1) / kThreads), kThreads, 0, st>>>((const float*)workspace, db, n, c,
                                                                                           (int)pl.tiles_adj);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}
