// Input of a super-res generator layer (generator_sres.py: Generator.prep_cond, the concatenation in
// SynthesisNetwork.forward and the cast at the start of SynthesisLayer.forward) as one op:
//
//   z[n', :C]        = dtype(x_prev[n'])                                     copy with cast
//   z[n', C + c S + s] = dtype(A_H L[n, c, t + s] A_W^T)                     n' = n T + t, S = window frames
//
// with A_H, A_W the per-axis plan of the layer's conditioning (torch_utils/ops/sres_cond.py builds it from the module's
// attributes): output index i -> resampler output m = x0 + clamp(i - px0, 0, mhi) (crop, then replicate pad), then the
// resampler's FIR out[m] = gain * sum_k f[K - 1 - k] * zu[m down + k - pad0] over the zero-upsampled (by `up`) replicate-
// padded frame, zero outside [0, zlen) (upfirdn2d's own zero padding), then sample v = j / up of that frame reads the
// low-res row / column clamp(v - shift, 0, len - 1) (the nested replicate pads). Identity axes: K = 0 (one tap of 1).
// The tap tables and both passes live in sres_cond.cuh: conv_pack_cond_kernel (conv_igemm.cu) evaluates the same sums.
//
// One launch: the first CTAs copy x_prev per sample (16-byte stores, loads as wide as the source's alignment allows,
// scalar head and tail), the rest each own a (n', channel, run of output rows) tile of the conditioning: per-axis tap
// tables and the vertical pass over the low-res frame (read through L1 / L2, element strides) are staged in shared
// memory, the horizontal pass writes z. With `sumsq`, every CTA also writes the sum of squares of the fp32 values of the
// concatenation (x before any cast, the conditioning before rounding) to one partial; a second kernel folds the partials
// in a fixed order into the mean. No atomics: bitwise reproducible. 64-bit element indices.
#include <type_traits>

#include "common.cuh"
#include "sres_cond.cuh"

namespace lvg {
namespace {

using sres::Axis;
using sres::axis_taps;
using sres::read_axis;

constexpr int kThreads = 256;
constexpr int kVecPerThread = 4;             // 16-byte vectors per thread of a copy CTA
constexpr int kRows = 16;                    // output rows per conditioning CTA
constexpr int kSmemBytes = 48 * 1024;

struct CondParams {
    const void* x;
    const float* lr;
    void* z;
    double* part;
    int64_t s_n, s_c, s_t, s_h, s_w;         // element strides of lr
    int n, t, c, c_lr, window, cc;           // cc = c_lr * window
    int rows, row_tiles;
    int bps;                                 // copy CTAs per sample
    int64_t copy_ctas;
    Axis ah, aw;
};

template <class T> __device__ __forceinline__ float ld1(const T* p) { return to_acc(__ldg(p)); }

// V consecutive elements of T from p, with loads of W bytes (p is W-aligned)
template <class T, int V, int W>
__device__ __forceinline__ void load_vec(const T* p, float (&v)[V])
{
    constexpr int kBytes = V * (int)sizeof(T);
    constexpr int kW = W < kBytes ? W : kBytes;
    using Chunk = typename std::conditional<kW == 16, uint4, typename std::conditional<kW == 8, uint2,
                  typename std::conditional<kW == 4, unsigned, unsigned short>::type>::type>::type;
    union { Chunk c[kBytes / kW]; T e[V]; } buf;
#pragma unroll
    for (int k = 0; k < kBytes / kW; k++) buf.c[k] = __ldg(reinterpret_cast<const Chunk*>(p) + k);
#pragma unroll
    for (int k = 0; k < V; k++) v[k] = to_acc(buf.e[k]);
}

template <class T, int V>
__device__ __forceinline__ void store_vec(T* p, const float (&v)[V])
{
    union { uint4 c; T e[V]; } buf;
#pragma unroll
    for (int k = 0; k < V; k++) buf.e[k] = from_acc<T>(v[k]);
    *reinterpret_cast<uint4*>(p) = buf.c;
}

// sum over the CTA of each thread's v, in a fixed order; the result is valid in thread 0
__device__ __forceinline__ double cta_sum(float v)
{
    __shared__ float swarp[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) swarp[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int k = 0; k < kThreads / 32; k++) s += (double)swarp[k];
    return s;
}

template <class TI, class TO, int W>
__device__ __forceinline__ float copy_body(const TI* __restrict__ src, TO* __restrict__ dst, int64_t h0, int64_t v0, int64_t v1)
{
    constexpr int V = 16 / (int)sizeof(TO);
    float sq = 0.f;
    for (int64_t k = v0 + threadIdx.x; k < v1; k += kThreads) {
        const int64_t e = h0 + k * V;
        float v[V];
        load_vec<TI, V, W>(src + e, v);
#pragma unroll
        for (int q = 0; q < V; q++) sq += v[q] * v[q];
        store_vec<TO, V>(dst + e, v);
    }
    return sq;
}

template <class TI, class TO, bool SQ>
__device__ void copy_cta(const CondParams& p, int64_t b)
{
    constexpr int V = 16 / (int)sizeof(TO);
    const int64_t hw = (int64_t)p.ah.out * p.aw.out;
    const int64_t e_n = (int64_t)p.c * hw;
    const int64_t np = b / p.bps;
    const int part = (int)(b % p.bps);
    const TI* src = (const TI*)p.x + np * e_n;
    TO* dst = (TO*)p.z + np * (int64_t)(p.c + p.cc) * hw;
    int64_t h0 = (int64_t)(((16 - ((uintptr_t)dst & 15)) & 15) / sizeof(TO));
    if (h0 > e_n) h0 = e_n;
    const int64_t nv = (e_n - h0) / V;
    const int64_t v0 = (int64_t)part * kThreads * kVecPerThread;
    const int64_t v1 = min(v0 + (int64_t)kThreads * kVecPerThread, nv);
    float sq = 0.f;
    const unsigned mis = (unsigned)((uintptr_t)(src + h0) & 15);
    if (mis == 0) sq = copy_body<TI, TO, 16>(src, dst, h0, v0, v1);
    else if ((mis & 7) == 0) sq = copy_body<TI, TO, 8>(src, dst, h0, v0, v1);
    else if ((mis & 3) == 0) sq = copy_body<TI, TO, 4>(src, dst, h0, v0, v1);
    else sq = copy_body<TI, TO, 2>(src, dst, h0, v0, v1);
    // scalar head (first CTA of the sample) and tail (last CTA)
    if (part == 0)
        for (int64_t e = threadIdx.x; e < h0; e += kThreads) {
            const float v = ld1(src + e);
            sq += v * v;
            dst[e] = from_acc<TO>(v);
        }
    if (part == p.bps - 1)
        for (int64_t e = h0 + nv * V + threadIdx.x; e < e_n; e += kThreads) {
            const float v = ld1(src + e);
            sq += v * v;
            dst[e] = from_acc<TO>(v);
        }
    if (SQ) {
        const double s = cta_sum(sq);
        if (threadIdx.x == 0) p.part[blockIdx.x] = s;
    }
}

template <class TO, bool SQ>
__device__ void cond_cta(const CondParams& p, int64_t b, unsigned char* smem)
{
    const int tile = (int)(b % p.row_tiles);
    const int64_t plane = b / p.row_tiles;
    const int ch = (int)(plane % p.cc);
    const int64_t np = plane / p.cc;
    const int n = (int)(np / p.t), t = (int)(np % p.t);
    const int c = ch / p.window, s = ch % p.window;
    const int r0 = tile * p.rows;
    const int rows = min(p.rows, p.ah.out - r0);
    const int wout = p.aw.out, wl = p.aw.len;
    const int nth = p.ah.nt, ntw = p.aw.nt;

    float* inter = reinterpret_cast<float*>(smem);                       // [rows][wl]
    float* wh = inter + p.rows * wl;                                     // [rows][nth]
    float* ww = wh + p.rows * nth;                                       // [wout][ntw]
    int* sh = reinterpret_cast<int*>(ww + wout * ntw);                   // [rows][nth]
    int* sw = sh + p.rows * nth;                                         // [wout][ntw]

    for (int r = threadIdx.x; r < rows; r += kThreads) axis_taps(p.ah, r0 + r, sh + r * nth, wh + r * nth);
    for (int i = threadIdx.x; i < wout; i += kThreads) axis_taps(p.aw, i, sw + i * ntw, ww + i * ntw);
    __syncthreads();

    // vertical pass: inter[r][x] = sum_k wh[r][k] L[sh[r][k]][x]
    const float* __restrict__ L = p.lr + n * p.s_n + c * p.s_c + (int64_t)(t + s) * p.s_t;
    for (int idx = threadIdx.x; idx < rows * wl; idx += kThreads) {
        const int r = idx / wl, x = idx - r * wl;
        inter[idx] = sres::vertical_tap_sum(L, p.s_h, p.s_w, x, wh + r * nth, sh + r * nth, nth);
    }
    __syncthreads();

    // horizontal pass: z = sum_k ww[i][k] inter[r][sw[i][k]]
    const int hout = p.ah.out;
    TO* __restrict__ out = (TO*)p.z + ((np * (p.c + p.cc) + p.c + ch) * hout + r0) * (int64_t)wout;
    float sq = 0.f;
    for (int idx = threadIdx.x; idx < rows * wout; idx += kThreads) {
        const int r = idx / wout, i = idx - r * wout;
        const float acc = sres::horizontal_tap_sum(inter + r * wl, ww + i * ntw, sw + i * ntw, ntw);
        sq += acc * acc;
        out[idx] = from_acc<TO>(acc);
    }
    if (SQ) {
        const double sum = cta_sum(sq);
        if (threadIdx.x == 0) p.part[blockIdx.x] = sum;
    }
}

template <class TI, class TO, bool SQ>
__global__ void __launch_bounds__(kThreads, 4) sres_cond_kernel(CondParams p)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int64_t b = blockIdx.x;
    if (b < p.copy_ctas) copy_cta<TI, TO, SQ>(p, b);
    else cond_cta<TO, SQ>(p, b - p.copy_ctas, smem);
}

// mean of the squares: the partials summed by one CTA in a fixed order
__global__ void __launch_bounds__(kThreads) sres_cond_fold_kernel(const double* __restrict__ part, int64_t nparts, double count,
                                                                  float* __restrict__ mean_sq)
{
    __shared__ double s[kThreads];
    double acc = 0.0;
    for (int64_t k = threadIdx.x; k < nparts; k += kThreads) acc += part[k];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *mean_sq = (float)(s[0] / count);
}

struct Plan {
    int rows, row_tiles, bps;
    int64_t copy_ctas, ctas;
    int smem;
};

bool make_plan(int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr, int z_dtype, const int* plan_h,
               const int* plan_w, Axis& ah, Axis& aw, Plan& pl)
{
    if (n < 1 || t < 1 || c < 0 || c_lr < 1 || window < 1 || h_lr < 1 || w_lr < 1 || !plan_h || !plan_w) return false;
    if (z_dtype != LVG_F32 && z_dtype != LVG_F16) return false;
    if ((int64_t)t + window - 1 > t_lr) return false;
    if (!read_axis(plan_h, h_lr, ah) || !read_axis(plan_w, w_lr, aw)) return false;
    const int64_t np = (int64_t)n * t, cc = (int64_t)c_lr * window;
    const int64_t hw = (int64_t)ah.out * aw.out;
    if ((np * (c + cc) * hw) >> 40) return false;
    pl.rows = ah.out < kRows ? ah.out : kRows;
    pl.row_tiles = (ah.out + pl.rows - 1) / pl.rows;
    const int64_t smem = ((int64_t)pl.rows * w_lr + 2ll * pl.rows * ah.nt + 2ll * aw.out * aw.nt) * 4;
    if (smem > kSmemBytes) return false;
    pl.smem = (int)smem;
    const int64_t e_n = (int64_t)c * hw;
    const int64_t vec = z_dtype == LVG_F32 ? 4 : 8, vec_per_cta = (int64_t)kThreads * kVecPerThread;
    const int64_t bps = (e_n / vec + vec_per_cta - 1) / vec_per_cta;              // covers every 16-byte vector of a sample
    pl.bps = c == 0 ? 0 : (int)(bps > 1 ? bps : 1);
    pl.copy_ctas = np * pl.bps;
    pl.ctas = pl.copy_ctas + np * cc * pl.row_tiles;
    return pl.ctas < (1ll << 31) - 1;
}

template <class TI, class TO>
int launch(const CondParams& p, const Plan& pl, float* mean_sq, double count, cudaStream_t st)
{
    if (mean_sq) sres_cond_kernel<TI, TO, true><<<(unsigned)pl.ctas, kThreads, pl.smem, st>>>(p);
    else sres_cond_kernel<TI, TO, false><<<(unsigned)pl.ctas, kThreads, pl.smem, st>>>(p);
    LVG_LAUNCH_CHECK();
    if (mean_sq) {
        sres_cond_fold_kernel<<<1, kThreads, 0, st>>>(p.part, pl.ctas, count, mean_sq);
        LVG_LAUNCH_CHECK();
    }
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_sres_cond_workspace(int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr, int z_dtype,
                                           const int* plan_h, const int* plan_w)
{
    Axis ah, aw;
    Plan pl;
    if (!make_plan(n, t, c, c_lr, window, t_lr, h_lr, w_lr, z_dtype, plan_h, plan_w, ah, aw, pl)) return LVG_UNSUPPORTED;
    return (pl.ctas * (int64_t)sizeof(double) + 15) & ~(int64_t)15;
}

extern "C" int lvg_sres_cond(const void* x, const float* lr, const float* f_h, const float* f_w, void* z, float* mean_sq,
                             void* workspace, int64_t workspace_bytes, int x_dtype, int z_dtype, int n, int t, int c, int c_lr,
                             int window, int t_lr, int h_lr, int w_lr, const int64_t* lr_strides, const int* plan_h,
                             const int* plan_w, float gain_h, float gain_w, void* stream)
{
    LVG_REQUIRE((x_dtype == LVG_F32 || x_dtype == LVG_F16) && (z_dtype == LVG_F32 || z_dtype == LVG_F16),
                "sres_cond: fp32 / fp16 only (x dtype %d, z dtype %d)", x_dtype, z_dtype);
    Axis ah, aw;
    Plan pl;
    if (!make_plan(n, t, c, c_lr, window, t_lr, h_lr, w_lr, z_dtype, plan_h, plan_w, ah, aw, pl)) {
        set_error("sres_cond: shape or plan outside the envelope (n %d t %d c %d, low-res %d x %d x %d x %d)", n, t, c, c_lr, t_lr,
                  h_lr, w_lr);
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(lr && z && lr_strides && (c == 0 || x), "sres_cond: lr, z and lr_strides (and x when c > 0) must not be NULL");
    LVG_REQUIRE((ah.ntaps == 0 || f_h) && (aw.ntaps == 0 || f_w), "sres_cond: a filtered axis needs its filter");
    LVG_REQUIRE(((uintptr_t)z % 16) == 0, "sres_cond: z must be 16-byte aligned");
    LVG_REQUIRE(c == 0 || ((uintptr_t)x % (x_dtype == LVG_F32 ? 4 : 2)) == 0, "sres_cond: x is not aligned to its element");
    if (mean_sq)
        LVG_REQUIRE(workspace && workspace_bytes >= pl.ctas * (int64_t)sizeof(double) && ((uintptr_t)workspace % 8) == 0,
                    "sres_cond: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                    (long long)(pl.ctas * (int64_t)sizeof(double)));
    ah.gain = gain_h; ah.f = f_h;
    aw.gain = gain_w; aw.f = f_w;
    CondParams p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.lr = lr; p.z = z; p.part = (double*)workspace;
    p.s_n = lr_strides[0]; p.s_c = lr_strides[1]; p.s_t = lr_strides[2]; p.s_h = lr_strides[3]; p.s_w = lr_strides[4];
    p.n = n; p.t = t; p.c = c; p.c_lr = c_lr; p.window = window; p.cc = c_lr * window;
    p.rows = pl.rows; p.row_tiles = pl.row_tiles; p.bps = pl.bps; p.copy_ctas = pl.copy_ctas;
    p.ah = ah; p.aw = aw;
    const double count = (double)n * t * (c + p.cc) * ah.out * (double)aw.out;
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == LVG_F32)
        return z_dtype == LVG_F32 ? launch<float, float>(p, pl, mean_sq, count, st) : launch<float, __half>(p, pl, mean_sq, count, st);
    return z_dtype == LVG_F32 ? launch<__half, float>(p, pl, mean_sq, count, st) : launch<__half, __half>(p, pl, mean_sq, count, st);
}
