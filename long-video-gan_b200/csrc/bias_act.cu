// bias_act: y = clamp(act(x + b) * gain) and its first / second derivatives.
//
// Semantics follow the reference kernel (torch_utils/ops/bias_act.cu:23-147):
// grad=0 evaluates the activation, grad=1 scales an incoming gradient by
// act'(.) expressed through the saved output yref (or the saved input xref for
// swish), grad=2 is the second derivative; clamping saturates in the forward
// and zeroes gradients where the forward output was saturated.
//
// Design: a pure streaming op (1 read + 1 write forward, 2 reads + 1 write
// backward), so the kernel is organised around bytes in flight: 128-bit
// loads/stores, four independent packs per thread issued before any use
// (64 KB in flight per SM at 4 CTAs/SM), grid sized in whole waves of the SM
// count, one bias lookup per 16-byte pack instead of a div+mod per element.
// The bias-gradient reduction can be fused into the backward pass
// (lvg_bias_act_grad_db) which removes the separate full read of dx.

#include "common.cuh"

namespace lvg {
namespace {

struct BiasActParams {
    const void* x;
    const void* b;
    const void* xref;
    const void* yref;
    const void* dy;
    void* y;
    float* db;        // fused bias-gradient accumulators (grad=1 only) or NULL
    uint8_t* codes;   // 2-bit sign / clamp codes (relu, lrelu): written by the forward pass, read INSTEAD of yref by the backward pass
    int64_t n;
    int64_t size_b;
    int64_t step_b;
    int run_tiles;    // fused db: consecutive tiles per run (see the kernel)
    uint64_t magic_step, magic_size;   // ceil(2^64 / d): exact quotients for operands < 2^32 (0 = divide for real)
    int grad;
    float alpha, gain, clamp;
};

// n / d through a multiply-high when the host could prepare a magic number (n, d < 2^32)
__device__ __forceinline__ int64_t fast_div(int64_t n, int64_t d, uint64_t magic)
{
    if (d == 1) return n;
    return magic ? (int64_t)__umul64hi((uint64_t)n, magic) : n / d;
}

// How the bias index of a 16-byte pack is obtained.
enum BiasMode {
    BIAS_NONE = 0,
    BIAS_PER_PACK = 1,   // step_b is a multiple of the pack width: one index per pack
    BIAS_PACKED = 2,     // step_b == 1 and size_b multiple of the pack width: load a bias pack
    BIAS_PER_ELEM = 3,   // anything else
};

__device__ __forceinline__ int64_t bias_row(int64_t elem, const BiasActParams& p) { return fast_div(elem, p.step_b, p.magic_step); }
__device__ __forceinline__ int64_t bias_index(int64_t elem, const BiasActParams& p)
{
    const int64_t row = bias_row(elem, p);
    return row - fast_div(row, p.size_b, p.magic_size) * p.size_b;
}

template <class S> __device__ __forceinline__ S fexp(S v);
template <> __device__ __forceinline__ float fexp<float>(float v) { return expf(v); }
template <> __device__ __forceinline__ double fexp<double>(double v) { return exp(v); }
template <class S> __device__ __forceinline__ S flog(S v);
template <> __device__ __forceinline__ float flog<float>(float v) { return logf(v); }
template <> __device__ __forceinline__ double flog<double>(double v) { return log(v); }
template <class S> __device__ __forceinline__ S ftanh(S v);
template <> __device__ __forceinline__ float ftanh<float>(float v) { return tanhf(v); }
template <> __device__ __forceinline__ double ftanh<double>(double v) { return tanh(v); }

// One element. `v` is x (grad 0) or the incoming gradient (grad>0); xr = xref + b;
// yr = yref; dyv = dy (grad 2) or 1.
template <class S, int A>
__device__ __forceinline__ S bias_act_elem(S v, S xr, S yr, S dyv, int G, S alpha, S gain, S inv_gain, S clamp)
{
    const S one = (S)1, two = (S)2;
    const S kExpRange = (S)80, kHalfExpRange = (S)40;
    const S kSeluScale = (S)1.0507009873554804934193349852946;
    const S kSeluAlpha = (S)1.6732632423543772848170429916717;
    const S r = yr * inv_gain;   // activation output before gain (inv_gain = 1/gain, 0 when gain is 0)
    S out = (S)0;

    if (A == LVG_ACT_LINEAR) {
        out = (G <= 1) ? v : (S)0;
    } else if (A == LVG_ACT_RELU) {
        if (G == 0) out = v > (S)0 ? v : (S)0;
        else if (G == 1) out = r > (S)0 ? v : (S)0;
    } else if (A == LVG_ACT_LRELU) {
        if (G == 0) out = v > (S)0 ? v : v * alpha;
        else if (G == 1) out = r > (S)0 ? v : v * alpha;
    } else if (A == LVG_ACT_TANH) {
        if (G == 0) out = ftanh(v);
        else if (G == 1) out = v * (one - r * r);
        else out = v * (one - r * r) * (-two * r);
    } else if (A == LVG_ACT_SIGMOID) {
        if (G == 0) out = (v < -kExpRange) ? (S)0 : one / (fexp(-v) + one);
        else if (G == 1) out = v * r * (one - r);
        else out = v * r * (one - r) * (one - two * r);
    } else if (A == LVG_ACT_ELU) {
        if (G == 0) out = (v >= (S)0) ? v : fexp(v) - one;
        else if (G == 1) out = (r >= (S)0) ? v : v * (r + one);
        else out = (r >= (S)0) ? (S)0 : v * (r + one);
    } else if (A == LVG_ACT_SELU) {
        if (G == 0) out = (v >= (S)0) ? kSeluScale * v : (kSeluScale * kSeluAlpha) * (fexp(v) - one);
        else if (G == 1) out = (r >= (S)0) ? v * kSeluScale : v * (r + kSeluScale * kSeluAlpha);
        else out = (r >= (S)0) ? (S)0 : v * (r + kSeluScale * kSeluAlpha);
    } else if (A == LVG_ACT_SOFTPLUS) {
        if (G == 0) out = (v > kExpRange) ? v : flog(fexp(v) + one);
        else if (G == 1) out = v * (one - fexp(-r));
        else { S c = fexp(-r); out = v * c * (one - c); }
    } else if (A == LVG_ACT_SWISH) {
        if (G == 0) {
            out = (v < -kExpRange) ? (S)0 : v / (fexp(-v) + one);
        } else {
            S c = fexp(xr);
            S d = c + one;
            if (G == 1) out = (xr > kHalfExpRange) ? v : v * c * (xr + d) / (d * d);
            else        out = (xr > kHalfExpRange) ? (S)0 : v * c * (xr * (two - d) + two * d) / (d * d * d);
            // swish keeps x, not y: rebuild the forward output for the clamp mask
            yr = (xr < -kExpRange) ? (S)0 : xr / (fexp(-xr) + one) * gain;
        }
    }

    out *= gain * dyv;

    if (clamp >= (S)0) {
        if (G == 0) out = (out > -clamp && out < clamp) ? out : (out >= (S)0 ? clamp : -clamp);
        else        out = (yr > -clamp && yr < clamp) ? out : (S)0;
    }
    return out;
}

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

template <class T>
__device__ __forceinline__ void fetch_bias(typename Acc<T>::type (&bias)[VecOf<T>::N], int64_t& bidx,
                                           const T* __restrict__ pb, int bmode, int64_t e0, const BiasActParams& p)
{
    typedef typename Acc<T>::type S;
    constexpr int N = VecOf<T>::N;
    bidx = 0;
    if (bmode == BIAS_PER_PACK) {
        bidx = bias_index(e0, p);
        S bv = pb ? to_acc(pb[bidx]) : (S)0;
#pragma unroll
        for (int k = 0; k < N; k++) bias[k] = bv;
    } else if (bmode == BIAS_PACKED) {
        bidx = e0 - fast_div(e0, p.size_b, p.magic_size) * p.size_b;
        Pack<T> vb;
        if (pb) vb = load_pack(pb + bidx);
#pragma unroll
        for (int k = 0; k < N; k++) bias[k] = pb ? to_acc(vb.v[k]) : (S)0;
    } else if (bmode == BIAS_PER_ELEM) {
#pragma unroll
        for (int k = 0; k < N; k++) bias[k] = pb ? to_acc(pb[bias_index(e0 + k, p)]) : (S)0;
    } else {
#pragma unroll
        for (int k = 0; k < N; k++) bias[k] = (S)0;
    }
}

// Vector kernel: n_pack packs of VecOf<T>::N elements, all operands 16-byte aligned.
// G is a template parameter so that grad 0 carries no reference operands at all.
// CODES: 0 = none; 1 = forward pass that also writes the 2-bit codes of its (stored) output: bit 0 "not positive",
// bit 1 "saturated by the clamp" -- everything the gradient of relu / lrelu depends on; 2 = backward pass that reads
// those codes instead of the saved output (1 byte per 16-byte fp32 pack, 2 per fp16 pack: the backward pass moves
// 2 n s + n / 4 bytes instead of 3 n s). The buffer is opaque to callers: a thread keeps the codes of the kUnroll packs
// it handles in a tile together (one 4- or 8-byte word at index tile * kThreads + thread), so both passes move them
// with one coalesced access per tile instead of kUnroll byte accesses.
template <class T, int A, int G, bool FUSE_DB, int CODES = 0>
__global__ void __launch_bounds__(kThreads, (G == 2 ? 2 : 4)) bias_act_vec_kernel(BiasActParams p, int64_t n_pack, int bmode)
{
    typedef typename Acc<T>::type S;
    constexpr int N = VecOf<T>::N;
    static_assert(CODES == 0 || ((A == LVG_ACT_RELU || A == LVG_ACT_LRELU) && (CODES == 1 ? G == 0 : G == 1)), "codes: relu / lrelu, forward writes, first-order backward reads");
    constexpr bool kUseX = (G > 0) && (A == LVG_ACT_SWISH);       // saved input
    constexpr bool kUseY = (G > 0) && (A != LVG_ACT_SWISH) && CODES != 2;       // saved output
    constexpr bool kUseDy = (G == 2);
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const S inv_gain = gain != (S)0 ? (S)1 / gain : (S)0;
    const T* __restrict__ px = (const T*)p.x;
    const T* __restrict__ pb = (const T*)p.b;
    const T* __restrict__ pxr = kUseX ? (const T*)p.xref : nullptr;
    const T* __restrict__ pyr = kUseY ? (const T*)p.yref : nullptr;
    const T* __restrict__ pdy = kUseDy ? (const T*)p.dy : nullptr;
    T* __restrict__ py = (T*)p.y;

    // Fused bias gradient (FUSE_DB): the tiles are walked in RUNS of p.run_tiles (8) consecutive tiles (128 KB of each operand; two
    // resident waves of CTAs), runs interleaved over the CTAs like single tiles are in the forward pass -- concurrently resident CTAs stream
    // one contiguous window of memory, which HBM rewards (single interleaved tiles with one atomic per warp and tile
    // serialise: ~100 consecutive tiles share a bias row and their atomics hit one address). Inside a run a warp stays inside one channel ("row" = run of
    // step_b elements sharing a bias index) for many packs: each lane keeps a running sum for the warp's current
    // row; only when the row changes or the run ends the warp reduces by shuffle and issues ONE global atomic.
    // No shared memory, no block barriers in the streaming loop.
    const int kRun = FUSE_DB ? p.run_tiles : 1;
    const int64_t tile = (int64_t)kThreads * kUnroll;
    const int64_t n_tiles = (n_pack + tile - 1) / tile;
    float run_sum = 0.f;           // this lane's share of the warp's current row
    int64_t run_row = -1, run_idx = 0;
    const unsigned full = 0xffffffffu;
    auto warp_flush = [&]() {
        float s = run_sum;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(full, s, o);
        if ((threadIdx.x & 31) == 0 && run_row >= 0) atomicAdd(p.db + run_idx, s);
        run_sum = 0.f;
    };

    for (int64_t run = blockIdx.x; run * kRun < n_tiles; run += gridDim.x) {
    const int64_t t_end = (run + 1) * kRun < n_tiles ? (run + 1) * kRun : n_tiles;
    for (int64_t t = run * kRun; t < t_end; t++) {
        const int64_t base = t * tile;
        Pack<T> vx[kUnroll], vref[kUnroll], vdy[kUnroll];
        unsigned vcode[kUnroll];
        const T* __restrict__ pref = kUseX ? pxr : pyr;
        uint2 cword = make_uint2(0u, 0u);            // this thread's codes of the tile: byte (fp32) / half-word (fp16) u = pack u
        if (CODES == 2) {
            if (N == 4) cword.x = __ldg(reinterpret_cast<const unsigned*>(p.codes) + t * kThreads + threadIdx.x);
            else cword = __ldg(reinterpret_cast<const uint2*>(p.codes) + t * kThreads + threadIdx.x);
        }
        // Bias along an outer dimension: almost every 16 KB tile lies inside ONE bias row (rows are ~100 tiles long in the
        // networks). Two divisions per tile (CTA-uniform) establish that; its packs then need no per-pack row arithmetic,
        // one bias value serves the whole tile, and the fused db needs no warp collectives.
        bool tile_one_row = false;
        int64_t tile_idx = 0;
        S tile_bias = (S)0;
        if (bmode == BIAS_PER_PACK) {
            const int64_t last = (base + tile < n_pack ? base + tile : n_pack) - 1;
            const int64_t r0 = bias_row(base * N, p), r1 = bias_row(last * N, p);
            tile_one_row = r0 == r1;
            if (tile_one_row) {
                tile_idx = r0 - fast_div(r0, p.size_b, p.magic_size) * p.size_b;
                if (pb) tile_bias = to_acc(pb[tile_idx]);
                if (FUSE_DB && r0 != run_row) {         // CTA-uniform, hence warp-uniform
                    warp_flush();
                    run_row = r0; run_idx = tile_idx;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const int64_t pk = base + (int64_t)u * kThreads + threadIdx.x;
            vcode[u] = (N == 4) ? (cword.x >> (8 * u)) & 0xffu : ((u < 2 ? cword.x : cword.y) >> (16 * (u & 1))) & 0xffffu;
            if (pk < n_pack) {
                vx[u] = load_pack(px + pk * N);

                if ((kUseX || kUseY) && pref) vref[u] = load_pack(pref + pk * N);
                if (kUseDy && pdy) vdy[u] = load_pack(pdy + pk * N);
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const int64_t pk = base + (int64_t)u * kThreads + threadIdx.x;
            int db_idx = -1;                    // tiles that straddle bias rows: this pack's bias index and sum
            float db_val = 0.f;
            if (pk < n_pack) {
                const int64_t e0 = pk * N;
                S bias[N];
                int64_t bidx;
                if (tile_one_row) {                     // bias index and value known for the whole tile
                    bidx = tile_idx;
#pragma unroll
                    for (int k = 0; k < N; k++) bias[k] = tile_bias;
                } else {
                    fetch_bias<T>(bias, bidx, pb, bmode, e0, p);
                }

                S fx[N], fref[N], fdy[N], fo[N];
                unpack<T>(vx[u], fx);
                if ((kUseX || kUseY) && pref) unpack<T>(vref[u], fref);
                if (kUseDy && pdy) unpack<T>(vdy[u], fdy);
#pragma unroll
                for (int k = 0; k < N; k++) {
                    S v = fx[k];
                    S xr = (kUseX && pref) ? fref[k] : (S)0;
                    S yr = (kUseY && pref) ? fref[k] : (S)0;
                    S dyv = (kUseDy && pdy) ? fdy[k] : (S)1;
                    if (G == 0) v += bias[k]; else xr += bias[k];
                    if (CODES == 2) {
                        // same arithmetic as the yref form: (not positive ? v * alpha | 0 : v) * gain, zero where the forward clamped
                        const unsigned cbits = vcode[u] >> (2 * k);
                        S o = (cbits & 1u) ? (A == LVG_ACT_LRELU ? v * alpha : (S)0) : v;
                        o *= gain;
                        fo[k] = (cbits & 2u) ? (S)0 : o;
                    } else {
                        fo[k] = bias_act_elem<S, A>(v, xr, yr, dyv, G, alpha, gain, inv_gain, clamp);
                    }
                }
                const Pack<T> out = pack<T>(fo);
                store_pack(py + e0, out);
                if (CODES == 1) {
                    // codes of what was STORED (after rounding to T), evaluated exactly like the backward pass evaluates yref:
                    // positive <=> yref * (1 / gain) > 0; saturated <=> not (-clamp < yref < clamp)
                    S ys[N];
                    if (sizeof(T) == sizeof(S)) {
#pragma unroll
                        for (int k = 0; k < N; k++) ys[k] = fo[k];
                    } else {
                        unpack<T>(out, ys);
                    }
                    unsigned code = 0;
                    if (inv_gain > (S)0) {          // the usual case (kernel-uniform): the sign of yref decides
#pragma unroll
                        for (int k = 0; k < N; k++) if (!(ys[k] > (S)0)) code |= 1u << (2 * k);
                    } else {
#pragma unroll
                        for (int k = 0; k < N; k++) if (!(ys[k] * inv_gain > (S)0)) code |= 1u << (2 * k);
                    }
                    if (clamp >= (S)0) {
#pragma unroll
                        for (int k = 0; k < N; k++) if (!(fabsf((float)ys[k]) < (float)clamp)) code |= 2u << (2 * k);
                    }
                    if (N == 4) cword.x |= code << (8 * u);
                    else if (u < 2) cword.x |= code << (16 * u);
                    else cword.y |= code << (16 * (u - 2));
                }
                if (FUSE_DB) {
                    // accumulate what was actually stored, like dx.sum() would see it
                    S fs[N];
                    unpack<T>(out, fs);
                    if (bmode == BIAS_PER_PACK) {
                        S s = (S)0;
#pragma unroll
                        for (int k = 0; k < N; k++) s += fs[k];
                        if (tile_one_row) run_sum += (float)s;
                        else { db_idx = (int)bidx; db_val = (float)s; }
                    } else {
#pragma unroll
                        for (int k = 0; k < N; k++) atomicAdd(p.db + bias_index(e0 + k, p), (float)fs[k]);
                    }
                }
            }
            if (FUSE_DB && bmode == BIAS_PER_PACK && !tile_one_row) {
                // short rows (small tensors) or a row boundary inside the tile: the warp's 32 packs usually still share
                // one bias index -> shuffle-reduce and one atomic; otherwise one atomic per lane. No state is carried.
                const int idx0 = __shfl_sync(full, db_idx, 0);
                if (__all_sync(full, db_idx == idx0 || db_idx < 0)) {
                    float sred = db_val;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sred += __shfl_xor_sync(full, sred, o);
                    if ((threadIdx.x & 31) == 0 && idx0 >= 0) atomicAdd(p.db + idx0, sred);
                } else if (db_idx >= 0) {
                    atomicAdd(p.db + db_idx, db_val);
                }
            }
        }
        if (CODES == 1) {
            if (N == 4) reinterpret_cast<unsigned*>(p.codes)[t * kThreads + threadIdx.x] = cword.x;
            else reinterpret_cast<uint2*>(p.codes)[t * kThreads + threadIdx.x] = cword;
        }
    }
    if (FUSE_DB && bmode == BIAS_PER_PACK) { warp_flush(); run_row = -1; }
    }
}

// Scalar kernel: fp64, unaligned buffers, and the < one-pack tail of the vector kernel.
template <class T, int A, bool FUSE_DB>
__global__ void __launch_bounds__(kThreads) bias_act_scalar_kernel(BiasActParams p, int64_t first)
{
    typedef typename Acc<T>::type S;
    const int G = p.grad;
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const S inv_gain = gain != (S)0 ? (S)1 / gain : (S)0;
    for (int64_t i = first + (int64_t)blockIdx.x * kThreads + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * kThreads) {
        S v = to_acc(((const T*)p.x)[i]);
        int64_t bidx = (p.b || FUSE_DB) ? bias_index(i, p) : 0;
        S bias = p.b ? to_acc(((const T*)p.b)[bidx]) : (S)0;
        S xr = p.xref ? to_acc(((const T*)p.xref)[i]) : (S)0;
        S yr = p.yref ? to_acc(((const T*)p.yref)[i]) : (S)0;
        S dyv = p.dy ? to_acc(((const T*)p.dy)[i]) : (S)1;
        if (G == 0) v += bias; else xr += bias;
        T o = from_acc<T>(bias_act_elem<S, A>(v, xr, yr, dyv, G, alpha, gain, inv_gain, clamp));
        ((T*)p.y)[i] = o;
        if (FUSE_DB) atomicAdd(p.db + bidx, (float)to_acc(o));
    }
}

// tuning knobs of the fused bias-gradient passes (environment overrides for experiments)
inline int fused_run_tiles() { static const int v = [] { const char* e = getenv("LVG_BA_RUN"); const int x = e ? atoi(e) : 0; return x >= 1 && x <= 64 ? x : 8; }(); return v; }
inline int fused_waves() { static const int v = [] { const char* e = getenv("LVG_BA_WAVES"); const int x = e ? atoi(e) : 0; return x >= 1 && x <= 16 ? x : 2; }(); return v; }

template <class T> struct HasVecPath { static constexpr bool value = true; };
template <> struct HasVecPath<double> { static constexpr bool value = false; };   // fp64 is a side path: scalar only

template <class T, int A, bool FUSE_DB>
int launch_typed(const BiasActParams& p, cudaStream_t stream)
{
    const int sms = num_sms();
    int64_t first = 0;

    if constexpr (HasVecPath<T>::value) {
        constexpr int N = VecOf<T>::N;
        const bool vec_ok = aligned16(p.x) && aligned16(p.y) && (!p.xref || aligned16(p.xref)) &&
                            (!p.yref || aligned16(p.yref)) && (!p.dy || aligned16(p.dy));
        const int64_t n_pack = vec_ok ? p.n / N : 0;
        if (n_pack > 0) {
            int mode = BIAS_NONE;
            if (p.b || FUSE_DB) {   // the fused db reduction needs the index even without bias values
                if (p.step_b % N == 0) mode = BIAS_PER_PACK;
                else if (p.step_b == 1 && p.size_b % N == 0 && (!p.b || aligned16(p.b))) mode = BIAS_PACKED;
                else mode = BIAS_PER_ELEM;
            }
            const int64_t tile = (int64_t)kThreads * kUnroll;
            int64_t blocks = (n_pack + tile - 1) / tile;
            // whole waves of 4 CTAs per SM; beyond 8 waves the grid-stride loop takes over
            int64_t cap = (int64_t)sms * 4 * 8;
            if (FUSE_DB) {          // runs of p.run_tiles tiles, whole resident waves so that every CTA gets ~the same number
                blocks = (blocks + p.run_tiles - 1) / p.run_tiles;
                cap = (int64_t)sms * 4 * fused_waves();
            }
            if (blocks > cap) blocks = cap;
            void (*k)(BiasActParams, int64_t, int) = nullptr;
            if (FUSE_DB)          k = bias_act_vec_kernel<T, A, 1, FUSE_DB>;
            else if (p.grad == 0) k = bias_act_vec_kernel<T, A, 0, false>;
            else if (p.grad == 1) k = bias_act_vec_kernel<T, A, 1, false>;
            else                  k = bias_act_vec_kernel<T, A, 2, false>;
            k<<<(unsigned)blocks, kThreads, 0, stream>>>(p, n_pack, mode);
            LVG_LAUNCH_CHECK();
        }
        first = n_pack * N;
    }
    if (first < p.n) {
        int64_t rest = p.n - first;
        int64_t blocks = (rest + kThreads - 1) / kThreads;
        const int64_t cap = (int64_t)sms * 8 * 4;
        if (blocks > cap) blocks = cap;
        bias_act_scalar_kernel<T, A, FUSE_DB><<<(unsigned)blocks, kThreads, 0, stream>>>(p, first);
        LVG_LAUNCH_CHECK();
    }
    return LVG_OK;
}

template <class T, bool FUSE_DB>
int launch_act(int act, const BiasActParams& p, cudaStream_t s)
{
    switch (act) {
        case LVG_ACT_LINEAR:   return launch_typed<T, LVG_ACT_LINEAR, FUSE_DB>(p, s);
        case LVG_ACT_RELU:     return launch_typed<T, LVG_ACT_RELU, FUSE_DB>(p, s);
        case LVG_ACT_LRELU:    return launch_typed<T, LVG_ACT_LRELU, FUSE_DB>(p, s);
        case LVG_ACT_TANH:     return launch_typed<T, LVG_ACT_TANH, FUSE_DB>(p, s);
        case LVG_ACT_SIGMOID:  return launch_typed<T, LVG_ACT_SIGMOID, FUSE_DB>(p, s);
        case LVG_ACT_ELU:      return launch_typed<T, LVG_ACT_ELU, FUSE_DB>(p, s);
        case LVG_ACT_SELU:     return launch_typed<T, LVG_ACT_SELU, FUSE_DB>(p, s);
        case LVG_ACT_SOFTPLUS: return launch_typed<T, LVG_ACT_SOFTPLUS, FUSE_DB>(p, s);
        case LVG_ACT_SWISH:    return launch_typed<T, LVG_ACT_SWISH, FUSE_DB>(p, s);
    }
    set_error("bias_act: unknown activation code %d", act);
    return LVG_ERR_ARG;
}

// relu / lrelu with 2-bit codes: forward (write = true) or first-order backward (optionally with the fused db)
template <class T, int A>
int launch_codes(const BiasActParams& p, bool write, bool fuse_db, cudaStream_t stream)
{
    constexpr int N = VecOf<T>::N;
    const bool vec_ok = aligned16(p.x) && aligned16(p.y) && (reinterpret_cast<uintptr_t>(p.codes) & 7) == 0 && p.n % N == 0;
    if (!vec_ok || (fuse_db && p.step_b % N != 0)) {
        set_error("bias_act codes: needs 16-byte aligned operands and a multiple of %d elements", N);
        return LVG_UNSUPPORTED;
    }
    const int64_t n_pack = p.n / N;
    int mode = BIAS_NONE;
    if (p.b || fuse_db) {
        if (p.step_b % N == 0) mode = BIAS_PER_PACK;
        else if (p.step_b == 1 && p.size_b % N == 0 && (!p.b || aligned16(p.b))) mode = BIAS_PACKED;
        else mode = BIAS_PER_ELEM;
    }
    const int64_t tile = (int64_t)kThreads * kUnroll;
    int64_t blocks = (n_pack + tile - 1) / tile;
    int64_t cap = (int64_t)num_sms() * 4 * 8;
    if (fuse_db) { blocks = (blocks + p.run_tiles - 1) / p.run_tiles; cap = (int64_t)num_sms() * 4 * fused_waves(); }
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    void (*k)(BiasActParams, int64_t, int) = write ? bias_act_vec_kernel<T, A, 0, false, 1>
                                           : fuse_db ? bias_act_vec_kernel<T, A, 1, true, 2> : bias_act_vec_kernel<T, A, 1, false, 2>;
    k<<<(unsigned)blocks, kThreads, 0, stream>>>(p, n_pack, mode);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

uint64_t magic_for(int64_t d, int64_t n)
{
    if (d <= 1 || d >= (1ll << 32) || n >= (1ll << 32)) return 0;
    return (uint64_t)(~0ull / (uint64_t)d) + 1;      // ceil(2^64 / d) for d that is not a power of two; exact enough otherwise too
}

int check_common(const void* x, const void* y, int dtype, int64_t n, const void* b, int64_t size_b, int64_t step_b, int act)
{
    LVG_REQUIRE(x && y, "bias_act: x and y must not be NULL");
    LVG_REQUIRE(dtype == LVG_F32 || dtype == LVG_F16 || dtype == LVG_F64, "bias_act: unsupported dtype %d", dtype);
    LVG_REQUIRE(n >= 0, "bias_act: negative element count");
    LVG_REQUIRE(!b || (size_b >= 1 && step_b >= 1), "bias_act: bias needs size_b >= 1 and step_b >= 1");
    LVG_REQUIRE(act >= LVG_ACT_LINEAR && act <= LVG_ACT_SWISH, "bias_act: unknown activation code %d", act);
    return LVG_OK;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int lvg_bias_act(const void* x, const void* b, const void* xref, const void* yref,
                            const void* dy, void* y, int dtype, int64_t n, int64_t size_b,
                            int64_t step_b, int grad, int act, float alpha, float gain,
                            float clamp, void* stream)
{
    int rc = check_common(x, y, dtype, n, b, size_b, step_b, act);
    if (rc) return rc;
    LVG_REQUIRE(grad >= 0 && grad <= 2, "bias_act: grad must be 0, 1 or 2 (got %d)", grad);
    if (n == 0) return LVG_OK;
    BiasActParams p = {x, b, xref, yref, dy, y, nullptr, nullptr, n, b ? size_b : 1, b ? step_b : 1, 1, 0, 0, grad, alpha, gain, clamp};
    p.magic_step = magic_for(p.step_b, n); p.magic_size = magic_for(p.size_b, n);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == LVG_F32) return launch_act<float, false>(act, p, s);
    if (dtype == LVG_F16) return launch_act<__half, false>(act, p, s);
    return launch_act<double, false>(act, p, s);
}

extern "C" int lvg_bias_act_grad_db(const void* dy_in, const void* b, const void* xref,
                                    const void* yref, void* dx, float* db_f32, int dtype,
                                    int64_t n, int64_t size_b, int64_t step_b, int act,
                                    float alpha, float gain, float clamp, void* stream)
{
    int rc = check_common(dy_in, dx, dtype, n, b, size_b, step_b, act);
    if (rc) return rc;
    LVG_REQUIRE(db_f32 != nullptr, "bias_act_grad_db: db buffer must not be NULL");
    LVG_REQUIRE(size_b >= 1 && step_b >= 1, "bias_act_grad_db: needs size_b >= 1 and step_b >= 1");
    LVG_REQUIRE(dtype == LVG_F32 || dtype == LVG_F16, "bias_act_grad_db: fp32/fp16 only");
    if (n == 0) return LVG_OK;
    // The fused reduction pays off when a 16-byte pack lies within one channel (bias along an outer
    // dimension). With the bias along the contiguous dimension (fully connected layers) every element
    // of a pack belongs to a different channel: leave that reduction to a separate pass.
    if (step_b % (dtype == LVG_F16 ? 8 : 4) != 0) {
        set_error("bias_act_grad_db: bias runs along the contiguous dimension; use bias_act(grad=1) + a reduction");
        return LVG_UNSUPPORTED;
    }
    // b may be NULL here (bias values are only needed by swish); the index math still applies.
    BiasActParams p = {dy_in, b, xref, yref, nullptr, dx, db_f32, nullptr, n, size_b, step_b, fused_run_tiles(), 0, 0, 1, alpha, gain, clamp};
    p.magic_step = magic_for(p.step_b, n); p.magic_size = magic_for(p.size_b, n);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == LVG_F32) return launch_act<float, true>(act, p, s);
    return launch_act<__half, true>(act, p, s);
}

extern "C" int lvg_bias_act_fwd_codes(const void* x, const void* b, void* y, void* codes, int dtype, int64_t n,
                                      int64_t size_b, int64_t step_b, int act, float alpha, float gain, float clamp,
                                      void* stream)
{
    int rc = check_common(x, y, dtype, n, b, size_b, step_b, act);
    if (rc) return rc;
    LVG_REQUIRE(codes != nullptr, "bias_act_fwd_codes: codes buffer must not be NULL");
    if ((act != LVG_ACT_RELU && act != LVG_ACT_LRELU) || (dtype != LVG_F32 && dtype != LVG_F16)) {
        set_error("bias_act_fwd_codes: relu / lrelu in fp32 / fp16 only");
        return LVG_UNSUPPORTED;
    }
    if (n == 0) return LVG_OK;
    BiasActParams p = {x, b, nullptr, nullptr, nullptr, y, nullptr, (uint8_t*)codes, n, b ? size_b : 1, b ? step_b : 1, 1, 0, 0, 0, alpha, gain, clamp};
    p.magic_step = magic_for(p.step_b, n); p.magic_size = magic_for(p.size_b, n);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == LVG_F32) return act == LVG_ACT_RELU ? launch_codes<float, LVG_ACT_RELU>(p, true, false, s) : launch_codes<float, LVG_ACT_LRELU>(p, true, false, s);
    return act == LVG_ACT_RELU ? launch_codes<__half, LVG_ACT_RELU>(p, true, false, s) : launch_codes<__half, LVG_ACT_LRELU>(p, true, false, s);
}

extern "C" int lvg_bias_act_bwd_codes(const void* dy, const void* codes, void* dx, float* db_f32, int dtype, int64_t n,
                                      int64_t size_b, int64_t step_b, int act, float alpha, float gain, float clamp,
                                      void* stream)
{
    int rc = check_common(dy, dx, dtype, n, nullptr, size_b, step_b, act);
    if (rc) return rc;
    LVG_REQUIRE(codes != nullptr, "bias_act_bwd_codes: codes buffer must not be NULL");
    LVG_REQUIRE(!db_f32 || (size_b >= 1 && step_b >= 1), "bias_act_bwd_codes: db needs size_b >= 1 and step_b >= 1");
    if ((act != LVG_ACT_RELU && act != LVG_ACT_LRELU) || (dtype != LVG_F32 && dtype != LVG_F16)) {
        set_error("bias_act_bwd_codes: relu / lrelu in fp32 / fp16 only");
        return LVG_UNSUPPORTED;
    }
    if (n == 0) return LVG_OK;
    const bool fuse = db_f32 != nullptr;
    BiasActParams p = {dy, nullptr, nullptr, nullptr, nullptr, dx, db_f32, (uint8_t*)codes, n, fuse ? size_b : 1, fuse ? step_b : 1, fused_run_tiles(), 0, 0, 1, alpha, gain, clamp};
    p.magic_step = magic_for(p.step_b, n); p.magic_size = magic_for(p.size_b, n);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == LVG_F32) return act == LVG_ACT_RELU ? launch_codes<float, LVG_ACT_RELU>(p, false, fuse, s) : launch_codes<float, LVG_ACT_LRELU>(p, false, fuse, s);
    return act == LVG_ACT_RELU ? launch_codes<__half, LVG_ACT_RELU>(p, false, fuse, s) : launch_codes<__half, LVG_ACT_LRELU>(p, false, fuse, s);
}

extern "C" int64_t lvg_bias_act_codes_bytes(int dtype, int64_t n)
{
    if (dtype != LVG_F32 && dtype != LVG_F16) return -1;
    const int pack = dtype == LVG_F16 ? 8 : 4;
    const int64_t tile = (int64_t)kThreads * kUnroll;
    const int64_t tiles = ((n + pack - 1) / pack + tile - 1) / tile;
    return tiles * kThreads * (dtype == LVG_F16 ? 8 : 4);
}
