// Super-res generator layer  y = d (.) conv(a (.) z, w)  with z = cat(x_prev, cond(lr)) never formed (DESIGN.md 7j): the
// re-tiling pass (conv_pack_cond_kernel) reads x_prev and evaluates the layer's conditioning from the low-res video by its
// plan (sres_cond.cuh: the tap tables and both passes of sres_cond_kernel, in the same order), rounds each value to the
// layer's dtype as lvg_sres_cond does, multiplies it by a and writes X8 as conv_pack_act_kernel does from z: bit for bit
// the modulated convolution of lvg_sres_cond's z. Channel c < C of a sample is x_prev's channel c, channel C + k window + s
// the conditioning of low-res channel k at frame t + s; a block of 8 channels may hold both.
// Backward: dgrad of d dy into all Cin channels (workspace), one streaming pass that dots each row with dtype(x_prev) or
// the conditioning (materialised for its c_lr window channels only, by lvg_sres_cond) for da and writes dx_prev =
// x_dtype(dtype(a dx')) for the x_prev channels, and the weight gradient from X8 rebuilt by the same re-tiling pass.
#include <algorithm>

#include "common.cuh"
#include "conv_engine.cuh"
#include "sres_cond.cuh"

namespace lvg {
namespace {

constexpr int kCondPackRows = 8;              // output rows per re-tiling CTA (shared memory: 8 channels x rows x low-res row)
constexpr int kCondPackSmem = 48 * 1024;

struct CondPackParams {
    const void* x;                            // x_prev [np][c][h][w] (TX), unused when c == 0
    const float* lr;
    uint4* y;                                 // X8 [np][nblk][h][w], or nullptr (SQ: only the sums of squares)
    const float* a;                           // [np][cin]
    double* part;                             // one sum of squares per CTA (SQ)
    int64_t s_n, s_c, s_t, s_h, s_w;          // element strides of lr
    int t, c, cin, window, cblk;
    int rows, row_tiles;
    sres::Axis ah, aw;
};

template <class TX, bool SPLIT, bool SQ>
__global__ void __launch_bounds__(256) conv_pack_cond_kernel(const CondPackParams p)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int64_t b = blockIdx.x;
    const int tile = (int)(b % p.row_tiles);
    const int blk = (int)((b / p.row_tiles) % p.cblk);
    const int64_t np = b / p.row_tiles / p.cblk;
    const int n = (int)(np / p.t), t = (int)(np % p.t);
    const int c0 = blk * 8;
    const int r0 = tile * p.rows;
    const int rows = min(p.rows, p.ah.out - r0);
    const int wout = p.aw.out, wl = p.aw.len;
    const int nth = p.ah.nt, ntw = p.aw.nt;
    // channels j < k0 of the block come from x_prev, k0 <= j < k1 from the conditioning, the rest are padding
    const int k0 = min(max(p.c - c0, 0), 8), k1 = min(max(p.cin - c0, 0), 8);

    float* inter = reinterpret_cast<float*>(smem);                       // [8][p.rows][wl]
    float* wh = inter + 8 * p.rows * wl;                                 // [p.rows][nth]
    float* ww = wh + p.rows * nth;                                       // [wout][ntw]
    int* sh = reinterpret_cast<int*>(ww + wout * ntw);                   // [p.rows][nth]
    int* sw = sh + p.rows * nth;                                         // [wout][ntw]
    if (k0 < k1) {                                                       // uniform over the CTA
        for (int r = threadIdx.x; r < rows; r += 256) sres::axis_taps(p.ah, r0 + r, sh + r * nth, wh + r * nth);
        for (int i = threadIdx.x; i < wout; i += 256) sres::axis_taps(p.aw, i, sw + i * ntw, ww + i * ntw);
        __syncthreads();
        const int plane = rows * wl;
        for (int idx = threadIdx.x; idx < (k1 - k0) * plane; idx += 256) {
            const int j = k0 + idx / plane, r = (idx % plane) / wl, x = idx % wl;
            const int ch = c0 + j - p.c, k = ch / p.window, s = ch % p.window;
            const float* __restrict__ L = p.lr + n * p.s_n + k * p.s_c + (int64_t)(t + s) * p.s_t;
            inter[(j * p.rows + r) * wl + x] = sres::vertical_tap_sum(L, p.s_h, p.s_w, x, wh + r * nth, sh + r * nth, nth);
        }
        __syncthreads();
    }

    const int64_t hw = (int64_t)p.ah.out * wout;
    const TX* __restrict__ xs = reinterpret_cast<const TX*>(p.x) + (np * p.c + c0) * hw;
    const float* __restrict__ as = p.a + np * p.cin + c0;
    const int nblk = SPLIT ? 2 * p.cblk : p.cblk;
    uint4* __restrict__ yo = p.y + (np * nblk + blk) * hw;
    float sq = 0.f;
    const bool store = p.y != nullptr;                                 // nullptr: the statistic alone
    for (int idx = threadIdx.x; idx < rows * wout; idx += 256) {
        const int r = idx / wout, i = idx - r * wout;
        const int64_t pix = (int64_t)(r0 + r) * wout + i;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            float f = 0.f;
            if (j < k0) f = to_acc(__ldg(xs + j * hw + pix));
            else if (j < k1) f = sres::horizontal_tap_sum(inter + (j * p.rows + r) * wl, ww + i * ntw, sw + i * ntw, ntw);
            if (SQ) sq += f * f;
            // the layer input z in the layer's dtype (lvg_sres_cond's rounding), then conv_pack_act_kernel's scaling
            if constexpr (!SPLIT) f = __half2float(__float2half_rn(f));
            v[j] = f;
        }
        if (!store) continue;
        if constexpr (!SPLIT) {
            alignas(16) unsigned short o[8];
#pragma unroll
            for (int j = 0; j < 8; j++) o[j] = j < k1 ? __half_as_ushort(__float2half_rn(v[j] * __ldg(as + j))) : (unsigned short)0;
            yo[pix] = *reinterpret_cast<const uint4*>(o);
        } else {
            alignas(16) unsigned short hi[8], lo[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const float f = j < k1 ? v[j] * __ldg(as + j) : 0.f;
                hi[j] = bf16_bits(f);
                lo[j] = bf16_bits(f - bf16_val(hi[j]));
            }
            yo[pix] = *reinterpret_cast<const uint4*>(hi);
            yo[(int64_t)p.cblk * hw + pix] = *reinterpret_cast<const uint4*>(lo);
        }
    }
    if (SQ) {
        __shared__ float swarp[8];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        if ((threadIdx.x & 31) == 0) swarp[threadIdx.x >> 5] = sq;
        __syncthreads();
        if (threadIdx.x == 0) {
            double s = 0.0;
            for (int k = 0; k < 8; k++) s += (double)swarp[k];
            p.part[blockIdx.x] = s;
        }
    }
}

// mean of the squares: the per-CTA partials summed by one CTA in a fixed order
__global__ void __launch_bounds__(256) conv_pack_cond_fold_kernel(const double* __restrict__ part, int64_t nparts, double count,
                                                                  float* __restrict__ mean_sq)
{
    __shared__ double s[256];
    double acc = 0.0;
    for (int64_t k = threadIdx.x; k < nparts; k += 256) acc += part[k];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *mean_sq = (float)(s[0] / count);
}

template <class T> __device__ __forceinline__ T round_to(float v);
template <> __device__ __forceinline__ float round_to<float>(float v) { return v; }
template <> __device__ __forceinline__ __half round_to<__half>(float v) { return __float2half_rn(v); }

// modconv_rowdot_kernel over the rows (sample, channel) of dx' [np][cin][len] (the layer's dtype T) against the layer input
// z without z: rows c < C read dtype(x_prev) (TX), the others the conditioning [np][cin - C][len] (T). da[row] = sum dx' z
// in modconv_rowdot_kernel's order; dx (NULL = not wanted) gets x_dtype(dtype(a dx')) for the x_prev rows.
template <class T, class TX, int VEC>
__global__ void __launch_bounds__(256) sres_layer_rowdot_kernel(const T* __restrict__ u, const TX* __restrict__ x, const T* __restrict__ cond,
                                                                const float* __restrict__ a, float* __restrict__ da, TX* __restrict__ dx,
                                                                int64_t rows, int cin, int c, int64_t len)
{
    __shared__ float red[8];
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        const int64_t np = row / cin;
        const int ch = (int)(row % cin);
        const bool from_x = ch < c;
        const T* ur = u + row * len;
        const TX* xr = x + (np * c + ch) * len;
        const T* cr = cond + (np * (cin - c) + (ch - c)) * len;
        TX* dr = dx + (np * c + ch) * len;
        const float sc = __ldg(a + row);
        float acc = 0.f;
        for (int64_t i = (int64_t)threadIdx.x * VEC; i < len; i += 256 * VEC) {
            alignas(16) T ue[VEC];
            if constexpr (VEC > 1) *reinterpret_cast<uint4*>(ue) = __ldg(reinterpret_cast<const uint4*>(ur + i));
            else ue[0] = ur[i];
#pragma unroll
            for (int j = 0; j < VEC; j++) {
                const float uf = to_f32(ue[j]);
                const float vf = from_x ? to_f32(round_to<T>(to_f32(__ldg(xr + i + j)))) : to_f32(__ldg(cr + i + j));
                acc += uf * vf;
                if (from_x && dx != nullptr) from_f32(dr[i + j], to_f32(round_to<T>(uf * sc)));
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int k = 0; k < 8; k++) s += red[k];
            da[row] = s;
        }
        __syncthreads();
    }
}

// one call of the layer op: the conditioning's shape and plan (as lvg_sres_cond takes them) and the convolution's
struct SresLayer {
    int n, t, c, c_lr, window, t_lr, h_lr, w_lr, cin, cout, kh, kw, pad_h, pad_w, dtype;
    int64_t np, hw;
    sres::Axis ah, aw;
    int rows, row_tiles, smem;
};

bool sres_layer_plan(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr, const int* plan_h, const int* plan_w,
                     int cout, int kh, int kw, int pad_h, int pad_w, SresLayer& L)
{
    if (n < 1 || t < 1 || c < 0 || c_lr < 1 || window < 1 || h_lr < 1 || w_lr < 1 || !plan_h || !plan_w) return false;
    if ((int64_t)t + window - 1 > t_lr || (int64_t)c + (int64_t)c_lr * window > (1 << 20)) return false;
    if (!sres::read_axis(plan_h, h_lr, L.ah) || !sres::read_axis(plan_w, w_lr, L.aw)) return false;
    L.n = n; L.t = t; L.c = c; L.c_lr = c_lr; L.window = window; L.t_lr = t_lr; L.h_lr = h_lr; L.w_lr = w_lr;
    L.cin = c + c_lr * window; L.cout = cout; L.kh = kh; L.kw = kw; L.pad_h = pad_h; L.pad_w = pad_w; L.dtype = dtype;
    L.np = (int64_t)n * t;
    L.hw = (int64_t)L.ah.out * L.aw.out;
    if ((L.np * std::max(L.cin, cout) * L.hw) >> 40) return false;
    if (!modconv_in_envelope({dtype, (int)std::min<int64_t>(L.np, 1 << 30), 1, L.cin, cout, 1, L.ah.out, L.aw.out, 1, kh, kw, 0, pad_h, pad_w, 1}))
        return false;
    if (L.np > (1 << 24)) return false;
    // the conditioning (and its per-call statistic) through lvg_sres_cond must take the same call
    if (lvg_sres_cond_workspace(n, t, 0, c_lr, window, t_lr, h_lr, w_lr, dtype, plan_h, plan_w) < 0) return false;
    for (L.rows = std::min(kCondPackRows, L.ah.out); L.rows >= 1; L.rows--) {
        L.smem = (int)((8ll * L.rows * w_lr + 2ll * L.rows * L.ah.nt + 2ll * L.aw.out * L.aw.nt) * 4);
        if (L.smem <= kCondPackSmem) break;
    }
    if (L.rows < 1) return false;
    L.row_tiles = (L.ah.out + L.rows - 1) / L.rows;
    return true;
}

int64_t sres_layer_pack_ctas(const SresLayer& L, int cblk) { return L.np * cblk * L.row_tiles; }

int sres_layer_pack(const SresLayer& L, const void* x, int x_dtype, const float* lr, const int64_t* st, const float* f_h, float gain_h,
                    const float* f_w, float gain_w, const float* a, void* x8, int cblk, double* part, cudaStream_t s)
{
    CondPackParams p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.lr = lr; p.y = (uint4*)x8; p.a = a; p.part = part;
    p.s_n = st[0]; p.s_c = st[1]; p.s_t = st[2]; p.s_h = st[3]; p.s_w = st[4];
    p.t = L.t; p.c = L.c; p.cin = L.cin; p.window = L.window; p.cblk = cblk;
    p.rows = L.rows; p.row_tiles = L.row_tiles;
    p.ah = L.ah; p.aw = L.aw;
    p.ah.f = f_h; p.ah.gain = gain_h;
    p.aw.f = f_w; p.aw.gain = gain_w;
    const int64_t ctas = sres_layer_pack_ctas(L, cblk);
    LVG_REQUIRE(ctas < (1ll << 31), "sres_layer: too many re-tiling CTAs");
    const bool split = L.dtype == LVG_F32, xf32 = x_dtype == LVG_F32, sq = part != nullptr;
    void (*const kerns[2][2][2])(const CondPackParams) = {
        {{conv_pack_cond_kernel<__half, false, false>, conv_pack_cond_kernel<__half, false, true>},
         {conv_pack_cond_kernel<__half, true, false>, conv_pack_cond_kernel<__half, true, true>}},
        {{conv_pack_cond_kernel<float, false, false>, conv_pack_cond_kernel<float, false, true>},
         {conv_pack_cond_kernel<float, true, false>, conv_pack_cond_kernel<float, true, true>}}};
    void (*kern)(const CondPackParams) = kerns[xf32][split][sq];
    kern<<<(unsigned)ctas, 256, L.smem, s>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

// the layer's convolution: every (sample, frame) an instance
ConvShape layer_shape(const SresLayer& L)
{
    return {L.dtype, (int)L.np, 1, L.cin, L.cout, 1, L.ah.out, L.aw.out, 1, L.kh, L.kw, 0, L.pad_h, L.pad_w, 1};
}

// workspace of the forward: [X8][the convolution's packed weights, as its job with X8 pre-tiled needs them][statistic partials]
struct SresLayerFwdRooms {
    int64_t x8, wp, part;
    int64_t total() const { return x8 + wp + part; }
};
SresLayerFwdRooms sres_layer_fwd_rooms(const SresLayer& L)
{
    const Geometry g = geometry(L.dtype == LVG_F32, L.np, 1, L.cin, L.cout, L.hw, L.kh * L.kw);
    const IgemmRooms c = igemm_rooms(fprop_job(layer_shape(L), nullptr, nullptr, nullptr));
    return {round256(c.x8), c.total() - c.x8, round256(sres_layer_pack_ctas(L, g.cblk) * (int64_t)sizeof(double))};
}

// workspace of the backward: [dx' over all Cin][conditioning][the convolution's backward]
struct SresLayerBwdRooms { int64_t dxp, cond, conv; };
SresLayerBwdRooms sres_layer_bwd_rooms(const SresLayer& L)
{
    const int es = L.dtype == LVG_F32 ? 4 : 2;
    return {round256(L.np * L.cin * L.hw * es), round256(L.np * (L.cin - L.c) * L.hw * es), backward_workspace(layer_shape(L))};
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_sres_layer_workspace(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                            const int* plan_h, const int* plan_w, int cout, int kh, int kw, int pad_h, int pad_w)
{
    SresLayer L;
    if (!sres_layer_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, kh, kw, pad_h, pad_w, L)) return -1;
    const SresLayerFwdRooms f = sres_layer_fwd_rooms(L);
    const SresLayerBwdRooms b = sres_layer_bwd_rooms(L);
    return std::max(f.total(), b.dxp + b.cond + b.conv);
}

extern "C" int lvg_sres_layer_fprop(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                                    const float* d, void* y, float* mean_sq, int x_dtype, int dtype, int n, int t, int c, int c_lr,
                                    int window, int t_lr, int h_lr, int w_lr, const int64_t* lr_strides, const int* plan_h,
                                    const int* plan_w, float gain_h, float gain_w, int cout, int kh, int kw, int pad_h, int pad_w,
                                    void* workspace, int64_t workspace_bytes, void* stream)
{
    SresLayer L;
    if (!sres_layer_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, kh, kw, pad_h, pad_w, L)) {
        set_error("sres_layer_fprop: shape, plan or convolution outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x_dtype == LVG_F32 || x_dtype == LVG_F16, "sres_layer_fprop: x_prev is fp32 or fp16");
    LVG_REQUIRE(lr && lr_strides && (c == 0 || x) && (y ? w && a : mean_sq != nullptr),
                "sres_layer_fprop: lr, lr_strides, x when c > 0, and w, a, y or (y NULL) mean_sq must not be NULL");
    LVG_REQUIRE((L.ah.ntaps == 0 || f_h) && (L.aw.ntaps == 0 || f_w), "sres_layer_fprop: a filtered axis needs its filter");
    LVG_REQUIRE(c == 0 || ((uintptr_t)x % (x_dtype == LVG_F32 ? 4 : 2)) == 0, "sres_layer_fprop: x is not aligned to its element");
    const SresLayerFwdRooms r = sres_layer_fwd_rooms(L);
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.total(), "sres_layer_fprop: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* x8 = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* wp = x8 + r.x8;
    double* part = mean_sq ? reinterpret_cast<double*>(wp + r.wp) : nullptr;
    const Geometry g = geometry(dtype == LVG_F32, L.np, 1, L.cin, cout, L.hw, kh * kw);
    int rc = sres_layer_pack(L, x, x_dtype, lr, lr_strides, f_h, gain_h, f_w, gain_w, a, y ? x8 : nullptr, g.cblk, part, s);
    if (rc) return rc;
    if (mean_sq) {
        conv_pack_cond_fold_kernel<<<1, 256, 0, s>>>(part, sres_layer_pack_ctas(L, g.cblk), (double)L.np * L.cin * (double)L.hw, mean_sq);
        LVG_LAUNCH_CHECK();
    }
    if (!y) return LVG_OK;
    IgemmJob j = fprop_job(layer_shape(L), nullptr, w, y);
    j.x8_pre = x8; j.out_scale = d;
    return run_igemm(j, wp, r.wp, s);
}

extern "C" int lvg_sres_layer_backward(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                                       const float* d, const void* y, const void* dy, void* dx, void* dw, float* da, float* dyy,
                                       int x_dtype, int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                       const int64_t* lr_strides, const int* plan_h, const int* plan_w, float gain_h, float gain_w,
                                       int cout, int kh, int kw, int pad_h, int pad_w, void* workspace, int64_t workspace_bytes,
                                       void* stream)
{
    SresLayer L;
    if (!sres_layer_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, kh, kw, pad_h, pad_w, L)) {
        set_error("sres_layer_backward: shape, plan or convolution outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x_dtype == LVG_F32 || x_dtype == LVG_F16, "sres_layer_backward: x_prev is fp32 or fp16");
    LVG_REQUIRE(lr && w && a && dy && da && lr_strides && (c == 0 || x), "sres_layer_backward: lr, w, a, dy, da, lr_strides (and x when c > 0) must not be NULL");
    LVG_REQUIRE(!dyy || (y && d), "sres_layer_backward: sum(dy * y) needs y and d");
    LVG_REQUIRE((L.ah.ntaps == 0 || f_h) && (L.aw.ntaps == 0 || f_w), "sres_layer_backward: a filtered axis needs its filter");
    LVG_REQUIRE(c == 0 || ((uintptr_t)x % (x_dtype == LVG_F32 ? 4 : 2)) == 0, "sres_layer_backward: x is not aligned to its element");
    const SresLayerBwdRooms r = sres_layer_bwd_rooms(L);
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.dxp + r.cond + r.conv,
                "sres_layer_backward: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    const int split = dtype == LVG_F32 ? 1 : 0;
    const ConvShape sh = layer_shape(L);
    const int np = (int)L.np;
    unsigned char* dxp = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* cond = dxp + r.dxp;
    unsigned char* conv = cond + r.cond;
    int rc;
    if (dyy) {
        rc = modconv_rowdot(const_cast<void*>(dy), y, nullptr, dyy, dtype, (int64_t)np * cout, (int64_t)sh.ho() * sh.wo(), s);
        if (rc) return rc;
    }
    // dx' = conv^T(d dy, w) over all Cin channels, as lvg_modconv_backward computes it
    Backward b;
    rc = backward_dgrad(sh, dy, d, w, dxp, conv, workspace_bytes - (r.dxp + r.cond), s, b);
    if (rc) return rc;
    // the conditioning channels of z, as lvg_sres_cond writes them
    rc = lvg_sres_cond(nullptr, lr, f_h, f_w, cond, nullptr, nullptr, 0, dtype, dtype, n, t, 0, c_lr, window, t_lr, h_lr, w_lr, lr_strides,
                       plan_h, plan_w, gain_h, gain_w, stream);
    if (rc) return rc;
    {
        const int64_t rows = (int64_t)np * L.cin, len = L.hw;
        const int64_t blocks = std::min<int64_t>(rows, (int64_t)num_sms() * 8);
        const bool vec = (len * (split ? 4 : 2)) % 16 == 0;
#define LVG_SRES_ROWDOT(T, TX, V)                                                                                                  \
    sres_layer_rowdot_kernel<T, TX, V><<<(unsigned)blocks, 256, 0, s>>>((const T*)dxp, (const TX*)x, (const T*)cond, a, da, (TX*)dx, rows, \
                                                                         L.cin, c, len)
        if (split) {
            if (x_dtype == LVG_F32) { if (vec) LVG_SRES_ROWDOT(float, float, 4); else LVG_SRES_ROWDOT(float, float, 1); }
            else { if (vec) LVG_SRES_ROWDOT(float, __half, 4); else LVG_SRES_ROWDOT(float, __half, 1); }
        } else {
            if (x_dtype == LVG_F32) { if (vec) LVG_SRES_ROWDOT(__half, float, 8); else LVG_SRES_ROWDOT(__half, float, 1); }
            else { if (vec) LVG_SRES_ROWDOT(__half, __half, 8); else LVG_SRES_ROWDOT(__half, __half, 1); }
        }
#undef LVG_SRES_ROWDOT
        LVG_LAUNCH_CHECK();
    }
    if (!dw) return LVG_OK;
    // dw from X8 of a z rebuilt by the re-tiling pass, in the slot the weight gradient would re-tile x into
    rc = sres_layer_pack(L, x, x_dtype, lr, lr_strides, f_h, gain_h, f_w, gain_w, a, b.x8, wgrad_plan(sh).cpad_b / 8, nullptr, s);
    if (rc) return rc;
    return backward_wgrad(sh, b, nullptr, dy, d, dw, nullptr, b.x8, s);
}
