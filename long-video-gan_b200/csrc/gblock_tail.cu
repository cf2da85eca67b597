// Tail of the low-res generator's residual block (Synthesis3dResBlock.forward, generator_lres.py:577-589) as one op:
//
//   m = (s + h) * sqrt(1/2)                          s: skip-convolution output, h: second modulated convolution output
//   u = crop_T(U_T m)       (U_T only with TUP)      2x linear upsampling, filter [1,3,3,1]/8, gain 2, padding (2, 1)
//   v = crop_HW(U_HW u)     (U_HW only with SUP)     the same filter on H and W, gain 4, padding (2, 1, 2, 1)
//   z = bias_act(v, b, lrelu | linear, clamp)
//
// Each upsampled axis is a polyphase 2-tap map: output position q = o + off (off = the centre crop's offset) reads input
// a = (q >> 1) - 1 + (q & 1) with weight 0.25 (q even) / 0.75 (q odd) and a + 1 with the complementary weight, taps
// outside the input reading zero -- exactly upfirdn2d.upsample2d's weights. Outputs are computed only at kept positions.
//
// Forward: a thread computes 4 consecutive elements of z. When the output rows are a multiple of 4 wide, the 4 outputs
// share a row: the thread sums s + h over its <= 2 x 2 (T, H) tap rows into a window of 4 input columns (one 128-bit load
// per row when the W axis is a plain aligned copy) and forms the 4 outputs from the window. It stores z once (128-bit for
// fp32) and, when a backward pass follows, one byte of 2-bit codes per 4 outputs in lvg_bias_act_fwd_codes' layout
// (bit 0 not positive, bit 1 clamped), evaluated on the stored value as bias_act evaluates them.
// Adjoint: dv = dz * gain * (lrelu slope | 1) * not clamped (from the codes), db = sum of dv, dm = sqrt(1/2) * the
// transposed upsamplings and crops applied to dv. A CTA owns a tile of m (one (n, c), a run of frames and rows, full
// width): it stages dv of every output its tile reaches in shared memory, evaluating each output once, sums dv over the
// outputs it owns (each output belongs to the tile of its first tap's input, so the tiles partition z), and gathers its
// tile of dm from shared memory. Each CTA writes one partial sum of db; a second kernel folds them per channel in a fixed
// order. No atomics: both directions are bitwise reproducible. 64-bit element indices throughout.
#include "common.cuh"

namespace lvg {
namespace {

constexpr int kThreads = 256;
constexpr int kAdjSmemBytes = 48 * 1024;
constexpr int kAdjTileElems = 4096;          // input elements a CTA's tile aims at
constexpr float kSqrtHalf = 0.70710678118654752440f;

struct TailParams {
    const void* s;
    const void* h;
    const float* b;
    void* z;
    uint8_t* codes;
    const void* dz;
    const uint8_t* codes_in;
    void* dm;
    float* part;
    int n, c, t, hh, ww, to, ho, wo;
    int off_t, off_h, off_w;
    int tup, sup;
    float alpha, gain, clamp;
    int64_t ne;                             // elements of z
    int tc, rc, n_tc, n_rc;                 // adjoint tiles: frames x rows per CTA, tiles per axis
};

// the two taps of output index o along an axis of `len` inputs: (i0, w0), (i1, w1); w = 0 for taps outside the input
__device__ __forceinline__ void taps2(int o, int off, int len, bool up, int& i0, float& w0, int& i1, float& w1)
{
    const int q = o + off;
    if (!up) { i0 = q; w0 = 1.f; i1 = q; w1 = 0.f; return; }
    i0 = (q >> 1) - 1 + (q & 1);
    i1 = i0 + 1;
    w0 = (q & 1) ? 0.75f : 0.25f;
    w1 = (q & 1) ? 0.25f : 0.75f;
    if (i0 < 0 || i0 >= len) w0 = 0.f;
    if (i1 < 0 || i1 >= len) w1 = 0.f;
}

template <class T> __device__ __forceinline__ float ldf(const T* p) { return to_acc(__ldg(p)); }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(__ldg(p)); }

// 4 consecutive elements from an address aligned to 4 elements
template <class T> __device__ __forceinline__ void load4(const T* p, float (&v)[4]);
template <> __device__ __forceinline__ void load4<float>(const float* p, float (&v)[4])
{
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
}
template <> __device__ __forceinline__ void load4<__half>(const __half* p, float (&v)[4])
{
    const uint2 q = __ldg(reinterpret_cast<const uint2*>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&q.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}

template <class T> __device__ __forceinline__ void store4(T* p, const float (&v)[4]);
template <> __device__ __forceinline__ void store4<float>(float* p, const float (&v)[4])
{
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void store4<__half>(__half* p, const float (&v)[4])
{
    const __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
    uint2 q;
    q.x = *reinterpret_cast<const unsigned*>(&a);
    q.y = *reinterpret_cast<const unsigned*>(&b);
    *reinterpret_cast<uint2*>(p) = q;
}

// byte of lvg_bias_act_fwd_codes' buffer that holds the codes of elements 4 g .. 4 g + 3: a thread of bias_act_vec_kernel
// keeps the codes of its kUnroll (4) packs of a 1024-pack tile in one word, byte (fp32) / half-word (fp16) u = pack u
template <class T> __device__ __forceinline__ int64_t code_byte(int64_t g)
{
    if (sizeof(T) == 4) {
        const int64_t pk = g;
        return (((pk >> 10) << 8) + (pk & 255)) * 4 + ((pk >> 8) & 3);
    }
    const int64_t pk = g >> 1;
    return (((pk >> 10) << 8) + (pk & 255)) * 8 + ((pk >> 8) & 3) * 2 + (g & 1);
}

// bias_act's forward of one element (bias_act_elem, grad 0) and the codes of the stored value
template <class T, int A>
__device__ __forceinline__ float activate(float v, const TailParams& p)
{
    float o = (A == LVG_ACT_LRELU) ? (v > 0.f ? v : v * p.alpha) : v;
    o *= p.gain;
    if (p.clamp >= 0.f) o = (o > -p.clamp && o < p.clamp) ? o : (o >= 0.f ? p.clamp : -p.clamp);
    return o;
}

template <class T>
__device__ __forceinline__ unsigned code_of(float y, const TailParams& p)
{
    const float ys = to_acc(from_acc<T>(y));
    const float inv_gain = p.gain != 0.f ? 1.f / p.gain : 0.f;
    unsigned code = (inv_gain > 0.f ? !(ys > 0.f) : !(ys * inv_gain > 0.f)) ? 1u : 0u;
    if (p.clamp >= 0.f && !(fabsf(ys) < p.clamp)) code |= 2u;
    return code;
}

// VEC: the output width is a multiple of 4, so a thread's 4 elements share one output row (window method); otherwise each
// element is decoded and gathered on its own.
template <class T, int A, bool VEC>
__global__ void __launch_bounds__(kThreads) gblock_tail_fwd_kernel(TailParams p)
{
    const T* __restrict__ ps = (const T*)p.s;
    const T* __restrict__ ph = (const T*)p.h;
    T* __restrict__ pz = (T*)p.z;
    const int64_t ngroups = (p.ne + 3) >> 2;
    const int64_t plane_in = (int64_t)p.t * p.hh * p.ww;
    const bool tup = p.tup, sup = p.sup;
    const bool linw = !sup && (p.ww & 3) == 0 && (p.off_w & 3) == 0;      // W is an aligned copy: 4-element loads

    for (int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x; g < ngroups; g += (int64_t)gridDim.x * kThreads) {
        const int64_t e0 = g << 2;
        float out[4];
        int nvalid = 4;
        if (VEC) {
            const int wo0 = (int)(e0 % p.wo);
            const int64_t row = e0 / p.wo;
            const int oh = (int)(row % p.ho);
            const int64_t r2 = row / p.ho;
            const int ot = (int)(r2 % p.to);
            const int64_t nc = r2 / p.to;
            const int ch = (int)(nc % p.c);
            int it[2], ih[2];
            float wt[2], wh[2];
            taps2(ot, p.off_t, p.t, tup, it[0], wt[0], it[1], wt[1]);
            taps2(oh, p.off_h, p.hh, sup, ih[0], wh[0], ih[1], wh[1]);
            // window of 4 input columns starting at ws; output k = win[ak] * wak + win[ak + 1] * wbk
            const int q0 = wo0 + p.off_w;
            const int ws = sup ? (q0 >> 1) - 1 + (q0 & 1) : q0;
            float win[4] = {0.f, 0.f, 0.f, 0.f};
            const int64_t base = nc * plane_in;
#pragma unroll
            for (int a = 0; a < 2; a++) {
                if (wt[a] == 0.f) continue;
#pragma unroll
                for (int bb = 0; bb < 2; bb++) {
                    if (wh[bb] == 0.f) continue;
                    const float wr = wt[a] * wh[bb];
                    const int64_t rb = base + ((int64_t)it[a] * p.hh + ih[bb]) * p.ww;
                    float sv[4], hv[4];
                    if (linw) {
                        load4<T>(ps + rb + ws, sv);
                        load4<T>(ph + rb + ws, hv);
                    } else {
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            const int col = ws + k;
                            const bool in = col >= 0 && col < p.ww;
                            sv[k] = in ? ldf(ps + rb + col) : 0.f;
                            hv[k] = in ? ldf(ph + rb + col) : 0.f;
                        }
                    }
#pragma unroll
                    for (int k = 0; k < 4; k++) win[k] += wr * (sv[k] + hv[k]);
                }
            }
            const float bias = p.b ? __ldg(p.b + ch) : 0.f;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                float v;
                if (sup) {
                    const int q = q0 + k;
                    const int ak = ((q >> 1) - 1 + (q & 1)) - ws;
                    const int col = ws + ak;
                    const float wa = (col >= 0 && col < p.ww) ? ((q & 1) ? 0.75f : 0.25f) : 0.f;
                    const float wb = (col + 1 >= 0 && col + 1 < p.ww) ? ((q & 1) ? 0.25f : 0.75f) : 0.f;
                    v = 0.f;
                    if (wa != 0.f) v += win[ak] * wa;
                    if (wb != 0.f) v += win[ak + 1] * wb;
                } else {
                    v = win[k];
                }
                out[k] = activate<T, A>(v * kSqrtHalf + bias, p);
            }
        } else {
            nvalid = p.ne - e0 < 4 ? (int)(p.ne - e0) : 4;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                out[k] = 0.f;
                if (k >= nvalid) continue;
                const int64_t e = e0 + k;
                const int ow = (int)(e % p.wo);
                const int64_t row = e / p.wo;
                const int oh = (int)(row % p.ho);
                const int64_t r2 = row / p.ho;
                const int ot = (int)(r2 % p.to);
                const int64_t nc = r2 / p.to;
                const int ch = (int)(nc % p.c);
                int it[2], ih[2], iw[2];
                float wt[2], wh[2], ww[2];
                taps2(ot, p.off_t, p.t, tup, it[0], wt[0], it[1], wt[1]);
                taps2(oh, p.off_h, p.hh, sup, ih[0], wh[0], ih[1], wh[1]);
                taps2(ow, p.off_w, p.ww, sup, iw[0], ww[0], iw[1], ww[1]);
                float acc = 0.f;
                for (int a = 0; a < 2; a++) {
                    if (wt[a] == 0.f) continue;
                    for (int bb = 0; bb < 2; bb++) {
                        if (wh[bb] == 0.f) continue;
                        const int64_t rb = nc * plane_in + ((int64_t)it[a] * p.hh + ih[bb]) * p.ww;
                        float rs = 0.f;
                        for (int cc = 0; cc < 2; cc++)
                            if (ww[cc] != 0.f) rs += ww[cc] * (ldf(ps + rb + iw[cc]) + ldf(ph + rb + iw[cc]));
                        acc += wt[a] * wh[bb] * rs;
                    }
                }
                const float bias = p.b ? __ldg(p.b + ch) : 0.f;
                out[k] = activate<T, A>(acc * kSqrtHalf + bias, p);
            }
        }
        if (nvalid == 4) {
            store4<T>(pz + e0, out);
        } else {
            for (int k = 0; k < nvalid; k++) pz[e0 + k] = from_acc<T>(out[k]);
        }
        if (p.codes) {
            unsigned byte = 0;
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (k < nvalid) byte |= code_of<T>(out[k], p) << (2 * k);
            p.codes[code_byte<T>(g)] = (uint8_t)byte;
        }
    }
}

// dv of z's element e from dz and the forward's codes (bias_act's first-order backward through the codes)
template <class T, int A>
__device__ __forceinline__ float dv_of(const T* __restrict__ pdz, const uint8_t* __restrict__ codes, int64_t e, const TailParams& p)
{
    const unsigned code = (__ldg(codes + code_byte<T>(e >> 2)) >> (2 * (e & 3))) & 3u;
    const float d = ldf(pdz + e);
    if (code & 2u) return 0.f;
    return ((A == LVG_ACT_LRELU && (code & 1u)) ? d * p.alpha : d) * p.gain;
}

// range of outputs [lo, hi) along an axis that the inputs [i0, i1) reach (reach = true: every tap) or own (first taps)
__device__ __forceinline__ void out_range(int i0, int i1, int off, int nout, bool up, bool reach, int& lo, int& hi)
{
    if (up) {
        lo = 2 * i0 - off - (reach ? 1 : 0);
        hi = 2 * i1 - off + (reach ? 1 : 0);
    } else {
        lo = i0 - off;
        hi = i1 - off;
    }
    lo = max(lo, 0);
    hi = min(hi, nout);
    if (hi < lo) hi = lo;
}

template <class T, int A>
__global__ void __launch_bounds__(kThreads) gblock_tail_adj_kernel(TailParams p)
{
    extern __shared__ float sdv[];
    __shared__ float swarp[kThreads / 32];
    const T* __restrict__ pdz = (const T*)p.dz;
    T* __restrict__ pdm = (T*)p.dm;
    const bool tup = p.tup, sup = p.sup;

    const int64_t blk = blockIdx.x;
    const int rcid = (int)(blk % p.n_rc);
    const int64_t r1 = blk / p.n_rc;
    const int tcid = (int)(r1 % p.n_tc);
    const int64_t nc = r1 / p.n_tc;
    const int i0 = tcid * p.tc, i1 = min(i0 + p.tc, p.t);
    const int j0 = rcid * p.rc, j1 = min(j0 + p.rc, p.hh);

    int ta, tb, ha, hb, ota, otb, oha, ohb;
    out_range(i0, i1, p.off_t, p.to, tup, true, ta, tb);
    out_range(j0, j1, p.off_h, p.ho, sup, true, ha, hb);
    out_range(i0, i1, p.off_t, p.to, tup, false, ota, otb);
    out_range(j0, j1, p.off_h, p.ho, sup, false, oha, ohb);
    const int nt = tb - ta, nh = hb - ha;

    // stage dv of every output the tile reaches; sum it over the outputs the tile owns
    float acc = 0.f;
    const int nstage = nt * nh * p.wo;
    for (int idx = threadIdx.x; idx < nstage; idx += kThreads) {
        const int ow = idx % p.wo;
        const int r = idx / p.wo;
        const int oh = ha + r % nh;
        const int ot = ta + r / nh;
        const int64_t e = ((nc * p.to + ot) * p.ho + oh) * (int64_t)p.wo + ow;
        const float d = dv_of<T, A>(pdz, p.codes_in, e, p);
        sdv[idx] = d;
        if (ot >= ota && ot < otb && oh >= oha && oh < ohb) acc += d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) swarp[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float sum = 0.f;
        for (int k = 0; k < kThreads / 32; k++) sum += swarp[k];
        p.part[blk] = sum;
    }

    // gather the tile of dm: input i receives from output positions 2i - 1 .. 2i + 2 with weights 1/4, 3/4, 3/4, 1/4
    const int rows = j1 - j0;
    const int ntile = (i1 - i0) * rows * p.ww;
    const int64_t plane_in = (int64_t)p.t * p.hh * p.ww;
    const float wq[4] = {0.25f, 0.75f, 0.75f, 0.25f};
    for (int idx = threadIdx.x; idx < ntile; idx += kThreads) {
        const int col = idx % p.ww;
        const int r = idx / p.ww;
        const int ih = j0 + r % rows;
        const int it = i0 + r / rows;
        float sum = 0.f;
        const int nqt = tup ? 4 : 1, nqh = sup ? 4 : 1, nqw = sup ? 4 : 1;
        for (int a = 0; a < nqt; a++) {
            const int ot = (tup ? 2 * it - 1 + a : it) - p.off_t;
            if (ot < 0 || ot >= p.to) continue;
            const float wa = tup ? wq[a] : 1.f;
            for (int bb = 0; bb < nqh; bb++) {
                const int oh = (sup ? 2 * ih - 1 + bb : ih) - p.off_h;
                if (oh < 0 || oh >= p.ho) continue;
                const float* srow = sdv + ((ot - ta) * nh + (oh - ha)) * p.wo;
                float rs = 0.f;
                for (int cc = 0; cc < nqw; cc++) {
                    const int ow = (sup ? 2 * col - 1 + cc : col) - p.off_w;
                    if (ow < 0 || ow >= p.wo) continue;
                    rs += (sup ? wq[cc] : 1.f) * srow[ow];
                }
                sum += wa * (sup ? wq[bb] : 1.f) * rs;
            }
        }
        pdm[nc * plane_in + ((int64_t)it * p.hh + ih) * p.ww + col] = from_acc<T>(sum * kSqrtHalf);
    }
}

// db[c] = sum over n and tiles of the CTAs' partial sums, in a fixed order
__global__ void __launch_bounds__(kThreads) gblock_tail_fold_kernel(const float* __restrict__ part, float* __restrict__ db, int n,
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
    int off_t, off_h, off_w;
    int tc, rc, n_tc, n_rc;
    int smem;
    int64_t ctas;
};

// offsets of the centre crops and the adjoint's tiling; false when the shape is outside the op's envelope
bool make_plan(int n, int c, int t, int h, int w, int to, int ho, int wo, int flags, Plan& pl)
{
    if (n < 1 || c < 1 || t < 1 || h < 1 || w < 1 || to < 1 || ho < 1 || wo < 1 || (flags & ~3)) return false;
    const bool tup = flags & LVG_GBLOCK_TAIL_TUP, sup = flags & LVG_GBLOCK_TAIL_SUP;
    const int64_t tu = tup ? 2ll * t : t, hu = sup ? 2ll * h : h, wu = sup ? 2ll * w : w;
    if (to > tu || ho > hu || wo > wu || tu > (1 << 30) || hu > (1 << 30) || wu > (1 << 30)) return false;
    pl.off_t = (int)((tu - to) / 2);
    pl.off_h = (int)((hu - ho) / 2);
    pl.off_w = (int)((wu - wo) / 2);
    auto reach = [](int k, bool up, int nout) { const int64_t r = up ? 2ll * k + 2 : k; return r < nout ? r : (int64_t)nout; };
    auto bytes = [&](int tc, int rc) { return reach(tc, tup, to) * reach(rc, sup, ho) * wo * (int64_t)sizeof(float); };
    int rc = h, tc = 1;
    while (rc > 1 && bytes(1, rc) > kAdjSmemBytes) rc = (rc + 1) / 2;
    if (bytes(1, rc) > kAdjSmemBytes) return false;
    while (tc < t && bytes(2 * tc, rc) <= kAdjSmemBytes && 2ll * tc * rc * w <= kAdjTileElems) tc *= 2;
    pl.tc = tc;
    pl.rc = rc;
    pl.n_tc = (t + tc - 1) / tc;
    pl.n_rc = (h + rc - 1) / rc;
    pl.smem = (int)bytes(tc, rc);
    pl.ctas = (int64_t)n * c * pl.n_tc * pl.n_rc;
    return pl.ctas < (1ll << 31) - 1;
}

int check_act(int dtype, int act)
{
    LVG_REQUIRE(dtype == LVG_F32 || dtype == LVG_F16, "gblock_tail: fp32 / fp16 only (got dtype %d)", dtype);
    if (act != LVG_ACT_LRELU && act != LVG_ACT_LINEAR) {
        set_error("gblock_tail: lrelu / linear only (got activation %d)", act);
        return LVG_UNSUPPORTED;
    }
    return LVG_OK;
}

TailParams params_of(const Plan& pl, int n, int c, int t, int h, int w, int to, int ho, int wo, int flags, float alpha, float gain,
                     float clamp)
{
    TailParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.c = c; p.t = t; p.hh = h; p.ww = w; p.to = to; p.ho = ho; p.wo = wo;
    p.off_t = pl.off_t; p.off_h = pl.off_h; p.off_w = pl.off_w;
    p.tup = (flags & LVG_GBLOCK_TAIL_TUP) != 0;
    p.sup = (flags & LVG_GBLOCK_TAIL_SUP) != 0;
    p.alpha = alpha; p.gain = gain; p.clamp = clamp;
    p.ne = (int64_t)n * c * to * ho * wo;
    p.tc = pl.tc; p.rc = pl.rc; p.n_tc = pl.n_tc; p.n_rc = pl.n_rc;
    return p;
}

template <class T, int A>
int launch_fwd(const TailParams& p, cudaStream_t stream)
{
    const int64_t groups = (p.ne + 3) >> 2;
    int64_t blocks = (groups + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    if (p.wo % 4 == 0) gblock_tail_fwd_kernel<T, A, true><<<(unsigned)blocks, kThreads, 0, stream>>>(p);
    else gblock_tail_fwd_kernel<T, A, false><<<(unsigned)blocks, kThreads, 0, stream>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

template <class T, int A>
int launch_adj(const TailParams& p, const Plan& pl, float* db, cudaStream_t stream)
{
    gblock_tail_adj_kernel<T, A><<<(unsigned)pl.ctas, kThreads, pl.smem, stream>>>(p);
    LVG_LAUNCH_CHECK();
    gblock_tail_fold_kernel<<<(unsigned)((p.c + kThreads - 1) / kThreads), kThreads, 0, stream>>>(p.part, db, p.n, p.c,
                                                                                                  pl.n_tc * pl.n_rc);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_gblock_tail_workspace(int n, int c, int t, int h, int w, int t_out, int h_out, int w_out, int flags)
{
    Plan pl;
    if (!make_plan(n, c, t, h, w, t_out, h_out, w_out, flags, pl)) return LVG_UNSUPPORTED;
    return (pl.ctas * (int64_t)sizeof(float) + 15) & ~(int64_t)15;
}

extern "C" int lvg_gblock_tail(const void* s, const void* h, const float* b, void* z, uint8_t* codes, int dtype, int n, int c,
                               int t, int hh, int ww, int t_out, int h_out, int w_out, int flags, int act, float alpha,
                               float gain, float clamp, void* stream)
{
    int rc = check_act(dtype, act);
    if (rc) return rc;
    LVG_REQUIRE(s && h && z, "gblock_tail: s, h and z must not be NULL");
    Plan pl;
    if (!make_plan(n, c, t, hh, ww, t_out, h_out, w_out, flags, pl)) {
        set_error("gblock_tail: shape outside the envelope (n %d c %d t %d h %d w %d -> %d x %d x %d, flags %d)", n, c, t, hh, ww,
                  t_out, h_out, w_out, flags);
        return LVG_UNSUPPORTED;
    }
    const int align = dtype == LVG_F32 ? 16 : 8;
    LVG_REQUIRE(((uintptr_t)z % align) == 0 && ((uintptr_t)s % align) == 0 && ((uintptr_t)h % align) == 0,
                "gblock_tail: s, h and z must be %d-byte aligned", align);
    TailParams p = params_of(pl, n, c, t, hh, ww, t_out, h_out, w_out, flags, alpha, gain, clamp);
    p.s = s; p.h = h; p.b = b; p.z = z; p.codes = codes;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == LVG_F32) return act == LVG_ACT_LRELU ? launch_fwd<float, LVG_ACT_LRELU>(p, st) : launch_fwd<float, LVG_ACT_LINEAR>(p, st);
    return act == LVG_ACT_LRELU ? launch_fwd<__half, LVG_ACT_LRELU>(p, st) : launch_fwd<__half, LVG_ACT_LINEAR>(p, st);
}

extern "C" int lvg_gblock_tail_adjoint(const void* dz, const uint8_t* codes, void* dm, float* db, void* workspace,
                                       int64_t workspace_bytes, int dtype, int n, int c, int t, int hh, int ww, int t_out,
                                       int h_out, int w_out, int flags, int act, float alpha, float gain, void* stream)
{
    int rc = check_act(dtype, act);
    if (rc) return rc;
    LVG_REQUIRE(dz && codes && dm && db && workspace, "gblock_tail_adjoint: dz, codes, dm, db and workspace must not be NULL");
    Plan pl;
    if (!make_plan(n, c, t, hh, ww, t_out, h_out, w_out, flags, pl)) {
        set_error("gblock_tail_adjoint: shape outside the envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(workspace_bytes >= pl.ctas * (int64_t)sizeof(float), "gblock_tail_adjoint: workspace of %lld bytes, %lld needed",
                (long long)workspace_bytes, (long long)(pl.ctas * (int64_t)sizeof(float)));
    TailParams p = params_of(pl, n, c, t, hh, ww, t_out, h_out, w_out, flags, alpha, gain, -1.f);
    p.dz = dz; p.codes_in = codes; p.dm = dm; p.part = (float*)workspace;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == LVG_F32) return act == LVG_ACT_LRELU ? launch_adj<float, LVG_ACT_LRELU>(p, pl, db, st) : launch_adj<float, LVG_ACT_LINEAR>(p, pl, db, st);
    return act == LVG_ACT_LRELU ? launch_adj<__half, LVG_ACT_LRELU>(p, pl, db, st) : launch_adj<__half, LVG_ACT_LINEAR>(p, pl, db, st);
}
