// The low-res generator's ToRGB layer (DESIGN.md 7l) as one pass over its input:
//
//   u[o] = sum_c w[o][c] a[n][c][t] r(x[c])       per pixel, w = weight / sqrt(cin) [3][cin] fp32, a = style * gain fp32
//   y    = dtype(clamp(dtype(u) + dtype(b), +-clamp))   bias_act's linear path
//
// r() is the rounding of x.type(dtype): x is read once in its own dtype and rounded in registers, never cast or copied.
// The layer has 3 output channels, so there is nothing for the tensor cores; it moves cin input values per 3 outputs and
// is bound by HBM. A CTA owns a run of pixels of one (n, t) plane and keeps w a of that plane in shared memory; each
// thread owns 8 consecutive pixels and keeps the 3 x 8 accumulators in registers. x is read with 16-byte loads when every
// plane starts on a 16-byte boundary (h w a multiple of 8, pointers 16-byte aligned), with scalar loads otherwise.
//
// Without a gain (a magnitude-EMA update whose gain is not known yet) the forward writes u in fp32 and a per-CTA partial
// of sum r(x)^2, folded in a fixed order into one sum; the caller updates the EMA on the device and lvg_lres_torgb_finish
// writes y = dtype(clamp(dtype(gain u) + dtype(b))).
//
// The backward reads x, y and dy once and writes dx once (bias_act's rule: dy passes where -clamp < y < clamp):
//   dx = x_dtype(a (w^T dy'))                                per pixel
//   G[n t][o][c] = sum_p dy'[o] r(x[c]),  S[n t][o] = sum_p dy'[o]
//   da[n][c][t] = sum_o w[o][c] G[o][c],  dw = sum_{n t} a G,  db = sum_{n t} S
// Each CTA writes its sums to one partial; two small kernels fold them in a fixed order (no atomics: every gradient is
// bitwise reproducible).
#include <algorithm>

#include "common.cuh"

namespace lvg {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPix = 8;                       // pixels per thread
constexpr int kCout = 3;
constexpr int kMaxCin = 512;

struct LresParams {
    const void* x;                            // [n][cin][t][hw] (TX)
    const float* w;                           // [3][cin]
    const float* a;                           // [n][cin][t]
    const float* b;                           // [3]
    void* y;                                  // [n][3][t][hw] (T) or nullptr
    float* u;                                 // [n][3][t][hw] or nullptr
    const void* dy;                           // [n][3][t][hw] (T)
    void* dx;                                 // [n][cin][t][hw] (TX) or nullptr
    float* part;                              // per CTA: 1 float (forward) or 3 cin + 3 floats (backward)
    int cin, t, hw, runs, tiles, tile_runs;
    int vec;
    float clamp;                              // < 0: none
};

template <class T> __device__ __forceinline__ float rnd(float v);
template <> __device__ __forceinline__ float rnd<float>(float v) { return v; }
template <> __device__ __forceinline__ float rnd<__half>(float v) { return __half2float(__float2half_rn(v)); }

// kPix consecutive elements at p (n of them valid when not vec)
template <class T>
__device__ __forceinline__ void load_run(const T* __restrict__ p, bool vec, int n, float (&v)[kPix])
{
    if (vec) {
#pragma unroll
        for (int h = 0; h < kPix / VecOf<T>::N; h++) {
            float f[VecOf<T>::N];
            unpack<T>(load_pack(p + h * VecOf<T>::N), f);
#pragma unroll
            for (int k = 0; k < VecOf<T>::N; k++) v[h * VecOf<T>::N + k] = f[k];
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
#pragma unroll
        for (int h = 0; h < kPix / VecOf<T>::N; h++) {
            float f[VecOf<T>::N];
#pragma unroll
            for (int k = 0; k < VecOf<T>::N; k++) f[k] = v[h * VecOf<T>::N + k];
            store_pack(p + h * VecOf<T>::N, pack<T>(f));
        }
    } else {
#pragma unroll
        for (int k = 0; k < kPix; k++)
            if (k < n) p[k] = from_acc<T>(v[k]);
    }
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// bias_act's clamp (linear activation): values outside (-clamp, clamp) go to the nearer bound
__device__ __forceinline__ float clamp_act(float v, float clamp)
{
    if (clamp >= 0.f && !(v > -clamp && v < clamp)) v = v >= 0.f ? clamp : -clamp;
    return v;
}

// the CTA's plane, its run of this thread and the first pixel of that run
struct Run {
    int64_t plane;                            // n t + t
    int n, t, q0, nv;
    __device__ Run(const LresParams& p)
    {
        plane = blockIdx.x / p.tiles;
        const int tile = (int)(blockIdx.x % p.tiles);
        n = (int)(plane / p.t);
        t = (int)(plane % p.t);
        const int run = tile * p.tile_runs + (int)threadIdx.x;
        const bool live = (int)threadIdx.x < p.tile_runs && run < p.runs;
        q0 = live ? run * kPix : 0;
        nv = live ? min(kPix, p.hw - q0) : 0;
    }
    // element offset of channel c at the run's first pixel in a [n][C][t][hw] tensor
    __device__ __forceinline__ int64_t at(const LresParams& p, int channels, int c) const
    {
        return (((int64_t)n * channels + c) * p.t + t) * p.hw + q0;
    }
};

// the per-CTA fixed-order sum of one value per thread (warp shuffles, then the warps in order)
__device__ __forceinline__ float block_sum(float v, float* red)
{
    v = warp_sum(v);
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = v;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0)
        for (int k = 0; k < kWarps; k++) s += red[k];
    return s;
}

template <class TX, class T>
__global__ void __launch_bounds__(kThreads) lres_torgb_fprop_kernel(const LresParams p)
{
    extern __shared__ __align__(16) float smem_f[];
    float* wa = smem_f;                                          // [3][cin]: w a of the plane
    const Run r(p);
    for (int k = threadIdx.x; k < kCout * p.cin; k += kThreads) {
        const int c = k % p.cin;
        wa[k] = __ldg(p.w + k) * __ldg(p.a + ((int64_t)r.n * p.cin + c) * p.t + r.t);
    }
    __syncthreads();
    const bool vec = p.vec != 0;
    const TX* __restrict__ xs = reinterpret_cast<const TX*>(p.x) + r.at(p, p.cin, 0);
    const int64_t cs = (int64_t)p.t * p.hw;                      // channel stride
    // two interleaved sums (even / odd channel): half the depth of one running sum
    float acc[kCout][kPix], acc1[kCout][kPix], sq = 0.f;
#pragma unroll
    for (int o = 0; o < kCout; o++)
#pragma unroll
        for (int k = 0; k < kPix; k++) acc[o][k] = acc1[o][k] = 0.f;
    if (r.nv > 0) {
#pragma unroll 2
        for (int ch = 0; ch < p.cin; ch += 2) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                if (ch + h >= p.cin) break;
                float v[kPix];
                load_run(xs + (ch + h) * cs, vec, r.nv, v);
                const float w0 = wa[ch + h], w1 = wa[p.cin + ch + h], w2 = wa[2 * p.cin + ch + h];
                float (&s)[kCout][kPix] = h ? acc1 : acc;
#pragma unroll
                for (int k = 0; k < kPix; k++) {
                    const float z = rnd<T>(v[k]);
                    sq = fmaf(z, z, sq);
                    s[0][k] = fmaf(w0, z, s[0][k]);
                    s[1][k] = fmaf(w1, z, s[1][k]);
                    s[2][k] = fmaf(w2, z, s[2][k]);
                }
            }
        }
        float bias[kCout] = {0.f, 0.f, 0.f};                     // b is NULL when u is written
        if (!p.u)
#pragma unroll
            for (int o = 0; o < kCout; o++) bias[o] = rnd<T>(__ldg(p.b + o));
#pragma unroll
        for (int o = 0; o < kCout; o++) {
            float out[kPix];
#pragma unroll
            for (int k = 0; k < kPix; k++) {
                const float u = acc[o][k] + acc1[o][k];
                out[k] = p.u ? u : clamp_act(rnd<T>(u) + bias[o], p.clamp);
            }
            if (p.u) store_run(p.u + r.at(p, kCout, o), vec, r.nv, out);
            else store_run(reinterpret_cast<T*>(p.y) + r.at(p, kCout, o), vec, r.nv, out);
        }
    }
    if (p.part) {
        __shared__ float red[kWarps];
        const float s = block_sum(sq, red);
        if (threadIdx.x == 0) p.part[blockIdx.x] = s;
    }
}

// sum of the forward's per-CTA partials in a fixed order (strided per thread, then a tree), in double
__global__ void __launch_bounds__(256) lres_torgb_fold_sq_kernel(const float* __restrict__ part, int64_t ctas, float* __restrict__ out)
{
    __shared__ double red[256];
    double s = 0.0;
    for (int64_t k = threadIdx.x; k < ctas; k += 256) s += part[k];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = (float)red[0];
}

// y = dtype(clamp(dtype(gain u) + dtype(b))) with the gain read from device memory
template <class T>
__global__ void __launch_bounds__(256) lres_torgb_finish_kernel(const float* __restrict__ u, const float* __restrict__ gain,
                                                                const float* __restrict__ b, T* __restrict__ y, int64_t total,
                                                                int64_t plane, float clamp)
{
    const float g = __ldg(gain);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int o = (int)((i / plane) % kCout);
        y[i] = from_acc<T>(clamp_act(rnd<T>(g * u[i]) + rnd<T>(__ldg(b + o)), clamp));
    }
}

template <class TX, class T>
__global__ void __launch_bounds__(kThreads) lres_torgb_backward_kernel(const LresParams p)
{
    extern __shared__ __align__(16) float smem_b[];
    const int cin = p.cin, nq = 3 * cin + kCout;
    float* wf = smem_b;                                          // [3][cin]
    float* af = wf + kCout * cin;                                // [cin]
    float* red = af + cin;                                       // [kWarps][3 cin + 3]
    const Run r(p);
    for (int k = threadIdx.x; k < kCout * cin; k += kThreads) wf[k] = __ldg(p.w + k);
    for (int c = threadIdx.x; c < cin; c += kThreads) af[c] = __ldg(p.a + ((int64_t)r.n * cin + c) * p.t + r.t);
    __syncthreads();
    const bool vec = p.vec != 0;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int64_t cs = (int64_t)p.t * p.hw;

    // dy' of the run: dy where -clamp < y < clamp
    float g[kCout][kPix];
#pragma unroll
    for (int o = 0; o < kCout; o++) {
        if (r.nv > 0) {
            float yv[kPix];
            load_run(reinterpret_cast<const T*>(p.y) + r.at(p, kCout, o), vec, r.nv, yv);
            load_run(reinterpret_cast<const T*>(p.dy) + r.at(p, kCout, o), vec, r.nv, g[o]);
#pragma unroll
            for (int k = 0; k < kPix; k++)
                if (p.clamp >= 0.f && !(yv[k] > -p.clamp && yv[k] < p.clamp)) g[o][k] = 0.f;
        } else {
#pragma unroll
            for (int k = 0; k < kPix; k++) g[o][k] = 0.f;
        }
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kPix; k++) s += g[o][k];
        s = warp_sum(s);
        if (lane == 0) red[warp * nq + 3 * cin + o] = s;
    }

    const TX* __restrict__ xs = reinterpret_cast<const TX*>(p.x) + r.at(p, cin, 0);
    TX* dxs = p.dx ? reinterpret_cast<TX*>(p.dx) + r.at(p, cin, 0) : nullptr;
#pragma unroll 2
    for (int ch = 0; ch < cin; ch++) {
        float z[kPix];
        if (r.nv > 0) load_run(xs + ch * cs, vec, r.nv, z);
        else
#pragma unroll
            for (int k = 0; k < kPix; k++) z[k] = 0.f;
        const float a = af[ch], w0 = wf[ch], w1 = wf[cin + ch], w2 = wf[2 * cin + ch];
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, dxo[kPix];
#pragma unroll
        for (int k = 0; k < kPix; k++) {
            const float zk = rnd<T>(z[k]);
            s0 = fmaf(g[0][k], zk, s0);
            s1 = fmaf(g[1][k], zk, s1);
            s2 = fmaf(g[2][k], zk, s2);
            dxo[k] = a * fmaf(w2, g[2][k], fmaf(w1, g[1][k], w0 * g[0][k]));
        }
        if (dxs && r.nv > 0) store_run(dxs + ch * cs, vec, r.nv, dxo);
        s0 = warp_sum(s0);
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        if (lane == 0) {
            float* q = red + warp * nq;
            q[ch] = s0;
            q[cin + ch] = s1;
            q[2 * cin + ch] = s2;
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

// per plane: G and S summed over the plane's tiles in tile order (to sums), and da = sum_o w[o][c] G[o][c]
__global__ void __launch_bounds__(256) lres_torgb_fold_tiles_kernel(const float* __restrict__ part, const float* __restrict__ w,
                                                                    int64_t planes, int tiles, int cin, int t,
                                                                    float* __restrict__ sums, float* __restrict__ da)
{
    const int nq = 3 * cin + kCout;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= planes * (cin + 1)) return;
    const int64_t pl = idx / (cin + 1);
    const int c = (int)(idx % (cin + 1));
    const float* src = part + pl * tiles * nq;
    if (c < cin) {
        float d = 0.f;
        for (int o = 0; o < kCout; o++) {
            float acc = 0.f;
            for (int k = 0; k < tiles; k++) acc += src[(int64_t)k * nq + o * cin + c];
            sums[pl * nq + o * cin + c] = acc;
            d = fmaf(__ldg(w + o * cin + c), acc, d);
        }
        if (da) {
            const int64_t n = pl / t, tt = pl % t;
            da[(n * cin + c) * t + tt] = d;
        }
    } else {
        for (int o = 0; o < kCout; o++) {
            float acc = 0.f;
            for (int k = 0; k < tiles; k++) acc += src[(int64_t)k * nq + 3 * cin + o];
            sums[pl * nq + 3 * cin + o] = acc;
        }
    }
}

// dw [3][cin] = sum over planes of a G, db [3] = sum over planes of S: one CTA per value, planes strided over the
// threads and the threads' sums added in a fixed tree
__global__ void __launch_bounds__(256) lres_torgb_fold_planes_kernel(const float* __restrict__ sums, const float* __restrict__ a,
                                                                     int64_t planes, int cin, int t, float* __restrict__ dw,
                                                                     float* __restrict__ db)
{
    __shared__ float red[256];
    const int nq = 3 * cin + kCout;
    const int q = blockIdx.x;
    const int c = q % cin;
    float s = 0.f;
    for (int64_t pl = threadIdx.x; pl < planes; pl += 256) {
        const float v = sums[pl * nq + q];
        s += q < 3 * cin ? __ldg(a + ((pl / t) * cin + c) * t + pl % t) * v : v;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (q < 3 * cin) {
            if (dw) dw[q] = red[0];
        } else if (db) {
            db[q - 3 * cin] = red[0];
        }
    }
}

struct Lres {
    int64_t planes, ctas;
    int n, cin, t, hw, runs, tiles, tile_runs;
    int64_t smem_fwd, smem_bwd;
};

bool lres_plan(int x_dtype, int dtype, int n, int cin, int t, int h, int w, int cout, int kt, int kh, int kw, Lres& L)
{
    if ((x_dtype != LVG_F16 && x_dtype != LVG_F32) || (dtype != LVG_F16 && dtype != LVG_F32)) return false;
    if (cout != kCout || kt != 1 || kh != 1 || kw != 1) return false;
    if (n < 1 || t < 1 || h < 1 || w < 1 || cin < 1 || cin > kMaxCin) return false;
    const int64_t hw = (int64_t)h * w;
    if (hw >= (1 << 30) || ((int64_t)n * cin * t * hw) >> 40) return false;
    L.n = n; L.cin = cin; L.t = t; L.hw = (int)hw;
    L.planes = (int64_t)n * t;
    L.runs = (int)((hw + kPix - 1) / kPix);
    L.tiles = (L.runs + kThreads - 1) / kThreads;
    L.tile_runs = (L.runs + L.tiles - 1) / L.tiles;              // balanced tiles of at most kThreads runs
    L.ctas = L.planes * L.tiles;
    if (L.ctas >= (1ll << 31)) return false;
    L.smem_fwd = (int64_t)kCout * cin * 4;
    L.smem_bwd = ((int64_t)kCout * cin + cin + (int64_t)kWarps * (3 * cin + kCout)) * 4;
    return true;
}

int64_t round256(int64_t v) { return (v + 255) / 256 * 256; }

struct LresRooms {
    int64_t part, sums;
    int64_t total() const { return part + sums; }
};
LresRooms lres_rooms(const Lres& L)
{
    const int64_t nq = 3 * L.cin + kCout;
    return {round256(L.ctas * nq * 4), round256(L.planes * nq * 4)};
}

LresParams lres_params(const Lres& L, const void* x, const float* w, const float* a, float clamp, bool vec)
{
    LresParams p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.w = w; p.a = a;
    p.cin = L.cin; p.t = L.t; p.hw = L.hw; p.runs = L.runs; p.tiles = L.tiles; p.tile_runs = L.tile_runs;
    p.vec = vec && L.hw % kPix == 0;
    p.clamp = clamp;
    return p;
}

bool aligned_to(const void* p, int64_t bytes) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }
bool aligned16_or_null(const void* p) { return p == nullptr || aligned16(p); }

template <class K>
int launch_planes(K kern, const Lres& L, int64_t smem, const LresParams& p, cudaStream_t s)
{
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)L.ctas, kThreads, (size_t)smem, s>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_lres_torgb_workspace(int x_dtype, int dtype, int n, int cin, int t, int h, int w, int cout, int kt, int kh, int kw)
{
    Lres L;
    if (!lres_plan(x_dtype, dtype, n, cin, t, h, w, cout, kt, kh, kw, L)) return -1;
    return lres_rooms(L).total();
}

extern "C" int lvg_lres_torgb_fprop(const void* x, const float* w, const float* a, const float* b, void* y, float* u, float* sumsq,
                                    int x_dtype, int dtype, int n, int cin, int t, int h, int wd, int cout, float clamp,
                                    void* workspace, int64_t workspace_bytes, void* stream)
{
    Lres L;
    if (!lres_plan(x_dtype, dtype, n, cin, t, h, wd, cout, 1, 1, 1, L)) {
        set_error("lres_torgb_fprop: shape or dtype outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x && w && a && (y || u), "lres_torgb_fprop: x, w, a and one of y / u must not be NULL");
    LVG_REQUIRE(!(y && u), "lres_torgb_fprop: y and u are exclusive");
    LVG_REQUIRE(u || b, "lres_torgb_fprop: b must not be NULL when y is written");
    const int xs = x_dtype == LVG_F32 ? 4 : 2, es = dtype == LVG_F32 ? 4 : 2;
    LVG_REQUIRE(aligned_to(x, xs) && aligned_to(y, es) && aligned_to(u, 4), "lres_torgb_fprop: x, y or u is not aligned to its element");
    if (sumsq)
        LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= L.ctas * 4,
                    "lres_torgb_fprop: workspace too small or misaligned for the sum of squares");
    LresParams p = lres_params(L, x, w, a, clamp, aligned16(x) && aligned16_or_null(y) && aligned16_or_null(u));
    p.b = b; p.y = y; p.u = u;
    p.part = sumsq ? reinterpret_cast<float*>(workspace) : nullptr;
    cudaStream_t s = (cudaStream_t)stream;
    void (*const kerns[2][2])(const LresParams) = {
        {lres_torgb_fprop_kernel<__half, __half>, lres_torgb_fprop_kernel<__half, float>},
        {lres_torgb_fprop_kernel<float, __half>, lres_torgb_fprop_kernel<float, float>}};
    int rc = launch_planes(kerns[x_dtype == LVG_F32][dtype == LVG_F32], L, L.smem_fwd, p, s);
    if (rc || !sumsq) return rc;
    lres_torgb_fold_sq_kernel<<<1, 256, 0, s>>>(p.part, L.ctas, sumsq);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

extern "C" int lvg_lres_torgb_finish(const float* u, const float* gain, const float* b, void* y, int dtype, int n, int t, int h, int wd,
                                     float clamp, void* stream)
{
    Lres L;
    if (!lres_plan(LVG_F32, dtype, n, 1, t, h, wd, kCout, 1, 1, 1, L)) {
        set_error("lres_torgb_finish: shape or dtype outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(u && gain && b && y, "lres_torgb_finish: u, gain, b and y must not be NULL");
    const int64_t plane = (int64_t)t * L.hw, total = (int64_t)n * kCout * plane;
    const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 16);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == LVG_F32)
        lres_torgb_finish_kernel<float><<<blocks, 256, 0, s>>>(u, gain, b, (float*)y, total, plane, clamp);
    else
        lres_torgb_finish_kernel<__half><<<blocks, 256, 0, s>>>(u, gain, b, (__half*)y, total, plane, clamp);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

extern "C" int lvg_lres_torgb_backward(const void* x, const float* w, const float* a, const void* y, const void* dy, void* dx, float* dw,
                                       float* da, float* db, int x_dtype, int dtype, int n, int cin, int t, int h, int wd, int cout,
                                       float clamp, void* workspace, int64_t workspace_bytes, void* stream)
{
    Lres L;
    if (!lres_plan(x_dtype, dtype, n, cin, t, h, wd, cout, 1, 1, 1, L)) {
        set_error("lres_torgb_backward: shape or dtype outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x && w && a && y && dy, "lres_torgb_backward: x, w, a, y and dy must not be NULL");
    const int xs = x_dtype == LVG_F32 ? 4 : 2, es = dtype == LVG_F32 ? 4 : 2;
    LVG_REQUIRE(aligned_to(x, xs) && aligned_to(dx, xs) && aligned_to(y, es) && aligned_to(dy, es),
                "lres_torgb_backward: x, dx, y or dy is not aligned to its element");
    const LresRooms r = lres_rooms(L);
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.total(), "lres_torgb_backward: workspace too small or misaligned");
    LresParams p = lres_params(L, x, w, a, clamp, aligned16(x) && aligned16_or_null(dx) && aligned16(y) && aligned16(dy));
    p.y = const_cast<void*>(y); p.dy = dy; p.dx = dx;
    p.part = reinterpret_cast<float*>(workspace);
    float* sums = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + r.part);
    cudaStream_t s = (cudaStream_t)stream;
    void (*const kerns[2][2])(const LresParams) = {
        {lres_torgb_backward_kernel<__half, __half>, lres_torgb_backward_kernel<__half, float>},
        {lres_torgb_backward_kernel<float, __half>, lres_torgb_backward_kernel<float, float>}};
    int rc = launch_planes(kerns[x_dtype == LVG_F32][dtype == LVG_F32], L, L.smem_bwd, p, s);
    if (rc) return rc;
    const int64_t fold = L.planes * (cin + 1);
    lres_torgb_fold_tiles_kernel<<<(unsigned)((fold + 255) / 256), 256, 0, s>>>(p.part, w, L.planes, L.tiles, cin, t, sums, da);
    LVG_LAUNCH_CHECK();
    if (dw || db) {
        lres_torgb_fold_planes_kernel<<<3 * cin + kCout, 256, 0, s>>>(sums, a, L.planes, cin, t, dw, db);
        LVG_LAUNCH_CHECK();
    }
    return LVG_OK;
}
