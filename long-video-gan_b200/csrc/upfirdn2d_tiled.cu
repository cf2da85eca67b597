// Single-launch separable upfirdn2d: both passes of a separable FIR (or one pass when the filter
// only spans one axis, e.g. the [k, 1] temporal filters on [N, C, T, H*W] tensors) in ONE kernel.
// The intermediate of the two-pass scheme (torch_utils/ops/upfirdn2d.py:244-245 writes it to HBM)
// stays in shared memory, so HBM sees exactly x once and y once.
//
// Per axis the operator is one of
//   ID            no filter: out[o] = x[o - pad0]
//   UP<S, F>      zero-insertion by S, F taps (F % S == 0), no decimation
//   DOWN<S, F>    F taps, keep every S-th sample (S == 1: plain filtering)
// with the definition of upfirdn2d.cu in this directory. Combinations of up- and down-sampling on
// the same axis, filters that are not a multiple of the up factor, and fp64 go to the general kernel.
//
// One CTA = one TOW x TOH output tile of one (n, c) plane: load the input tile (zero outside the
// image) -> x pass into a second tile -> y pass straight to global memory. Tile sizes are chosen
// on the host per call (runtime), filter length and factors are template parameters so the taps
// live in registers and the polyphase loops unroll (fir_passes.cuh).

#include "common.cuh"
#include "fir_passes.cuh"

namespace lvg {

int upfirdn2d_check(const void* x, const void* y, int dtype, const int64_t* xsh, const int64_t* ysh,
                    int fw, int fh, int upx, int upy, int downx, int downy);
int upfirdn2d_stream(const void* x, const float* fx, int64_t fsx, const float* fy, int64_t fsy, void* y, int dtype,
                     const int64_t* xsh, const int64_t* xst, const int64_t* ysh, const int64_t* yst,
                     int fw, int fh, int upx, int upy, int downx, int downy, int padx0, int pady0,
                     int flip, float gain, cudaStream_t s);

namespace {

enum { AX_ID = 0, AX_UP = 1, AX_DOWN = 2 };

struct TiledParams {
    const void* x;
    const float* fx;
    const float* fy;
    void* y;
    int64_t xs[4], ys[4];
    int64_t fsx, fsy;     // element strides of the tap vectors
    int n, c, ih, iw, oh, ow;
    int padx0, pady0;
    int flip;
    float gain;
    int tow, toh, tiles_x, tiles_y;
    int pb;               // planes per CTA (> 1 only when one tile covers the whole plane)
    int flat;             // 1: the CTA's input planes are one contiguous, 16-byte aligned block (vector loader);
                          // 2: additionally every input element lies inside the tile (no bounds checks)
    fir::FastDiv by_plane_elems, by_iw;   // host-made dividers of the vector loader
    int64_t planes;       // n * c
    int p_in, p_mid;      // row pitches (odd)
    int a_size;           // floats reserved for the input tile(s)
};

constexpr int kThreads = 256;
constexpr int kR = 4;

// extent of the input tile an axis needs for `n` outputs (upper bound over alignments)
template <int KIND, int S, int F>
__host__ __device__ constexpr int in_extent(int n)
{
    return KIND == AX_ID ? n
         : KIND == AX_DOWN ? (fir::round_up(n, kR) - 1) * S + F
         : fir::round_up((n + S - 1 + S - 1) / S, kR) + F / S;
}
// extent of the x-pass output (row length of the mid tile)
template <int KIND, int S, int F>
__host__ __device__ constexpr int mid_extent(int n)
{
    return KIND == AX_UP ? fir::round_up((n + S - 1 + S - 1) / S, kR) * S : fir::round_up(n, kR);
}


// ---- y passes that store straight to global memory.
// Paired like the x passes of fir_passes.cuh, but along columns: lane L owns columns L and L + 32 of a 64-column span,
// R groups / outputs along y per item. The store addresses are formed ONCE per item as two 64-bit column
// pointers; every result then costs one pointer bump and one store, and items that lie completely inside the
// tile (all but the first / last along y) take a path without row checks. `ys*` are element strides of y; the
// host guarantees that one CTA's outputs span < 2^31 elements.
template <class T> __device__ __forceinline__ T* opaque(T* p)
{
    asm volatile("" : "+l"(p));      // keeps the compiler from re-deriving the pointer from its 64-bit offset form per store
    __builtin_assume(__isGlobal(p));
    return p;
}

template <class T, int UP, int F, int R, int NTHREADS>
__device__ __forceinline__ void up_y2_store(const float* __restrict__ in, int pin, int cols, int groups, const float* __restrict__ s_taps,
                                            T* yp, int ys1, int ys2, int ys3, int dyo, int toh_e, int nplanes, int plane_rows)
{
    constexpr int K = F / UP;
    float2 g[F];
#pragma unroll
    for (int i = 0; i < F; i++) g[i] = make_float2(s_taps[i], s_taps[i]);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int gthreads = (groups + R - 1) / R;
    const int vcols = nplanes * cols;
    const int n_cc = (vcols + 63) / 64;
    const fir::FastDiv by_cols(cols), by_cc(n_cc);
    for (int wi = warp; wi < gthreads * n_cc; wi += NTHREADS / 32) {
        const int tg = by_cc.div(wi), cc = wi - tg * n_cc;
        const int va = cc * 64 + lane, vb = va + 32;
        if (va < vcols) {
            const bool has_b = vb < vcols;
            const int pla = nplanes > 1 ? by_cols.div(va) : 0, cola = va - pla * cols;
            const int plb = has_b ? (nplanes > 1 ? by_cols.div(vb) : 0) : pla, colb = has_b ? vb - plb * cols : cola;
            const float* sa = in + (pla * plane_rows + tg * R) * pin + cola;
            const float* sb = in + (plb * plane_rows + tg * R) * pin + colb;
            float2 v[K + R];
#pragma unroll
            for (int i = 0; i < K + R; i++) v[i] = make_float2(sa[i * pin], sb[i * pin]);
            const int o0 = tg * R * UP - dyo;                       // output row of the item's first result (may be < 0)
            T* pa = opaque(yp + (pla * ys1 + cola * ys3 + o0 * ys2));
            T* pb = opaque(yp + (plb * ys1 + colb * ys3 + o0 * ys2));
            const bool full = o0 >= 0 && o0 + R * UP <= toh_e;      // warp-uniform
            if (full) {
#pragma unroll
                for (int j = 0; j < R; j++) {
#pragma unroll
                    for (int ph = 0; ph < UP; ph++) {
                        float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                        for (int k = 0; k < K; k++) acc = fir::ffma2(g[(UP - ph) % UP + k * UP], v[j + (ph > 0 ? 1 : 0) + k], acc);
                        *pa = from_acc<T>(acc.x);
                        if (has_b) *pb = from_acc<T>(acc.y);
                        pa += ys2; pb += ys2;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < R; j++) {
#pragma unroll
                    for (int ph = 0; ph < UP; ph++) {
                        float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                        for (int k = 0; k < K; k++) acc = fir::ffma2(g[(UP - ph) % UP + k * UP], v[j + (ph > 0 ? 1 : 0) + k], acc);
                        if ((unsigned)(o0 + j * UP + ph) < (unsigned)toh_e) {
                            *pa = from_acc<T>(acc.x);
                            if (has_b) *pb = from_acc<T>(acc.y);
                        }
                        pa += ys2; pb += ys2;
                    }
                }
            }
        }
    }
}

template <class T, int DOWN, int F, int R, int NTHREADS>
__device__ __forceinline__ void down_y2_store(const float* __restrict__ in, int pin, int cols, int outs, const float* __restrict__ s_taps,
                                              T* yp, int ys1, int ys2, int ys3, int nplanes, int plane_rows)
{
    constexpr int NIN = (R - 1) * DOWN + F;
    float2 g[F];
#pragma unroll
    for (int i = 0; i < F; i++) g[i] = make_float2(s_taps[i], s_taps[i]);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int gthreads = (outs + R - 1) / R;
    const int vcols = nplanes * cols;
    const int n_cc = (vcols + 63) / 64;
    const fir::FastDiv by_cols(cols), by_cc(n_cc);
    for (int wi = warp; wi < gthreads * n_cc; wi += NTHREADS / 32) {
        const int tg = by_cc.div(wi), cc = wi - tg * n_cc;
        const int va = cc * 64 + lane, vb = va + 32;
        if (va < vcols) {
            const bool has_b = vb < vcols;
            const int pla = nplanes > 1 ? by_cols.div(va) : 0, cola = va - pla * cols;
            const int plb = has_b ? (nplanes > 1 ? by_cols.div(vb) : 0) : pla, colb = has_b ? vb - plb * cols : cola;
            const float* sa = in + (pla * plane_rows + tg * R * DOWN) * pin + cola;
            const float* sb = in + (plb * plane_rows + tg * R * DOWN) * pin + colb;
            float2 v[NIN];
#pragma unroll
            for (int i = 0; i < NIN; i++) v[i] = make_float2(sa[i * pin], sb[i * pin]);
            const int o0 = tg * R;
            T* pa = opaque(yp + (pla * ys1 + cola * ys3 + o0 * ys2));
            T* pb = opaque(yp + (plb * ys1 + colb * ys3 + o0 * ys2));
            const bool full = o0 + R <= outs;                       // warp-uniform
#pragma unroll
            for (int j = 0; j < R; j++) {
                float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                for (int t = 0; t < F; t++) acc = fir::ffma2(g[t], v[j * DOWN + t], acc);
                if (full || o0 + j < outs) {
                    *pa = from_acc<T>(acc.x);
                    if (has_b) *pb = from_acc<T>(acc.y);
                }
                pa += ys2; pb += ys2;
            }
        }
    }
}

template <class T, int KX, int SX, int FX, int KY, int SY, int FY>
__global__ void __launch_bounds__(kThreads) upfirdn2d_tiled_kernel(TiledParams p)
{
    extern __shared__ __align__(16) float smem[];
    // layout: [input tile a_size][mid tile (absent when the x axis is ID)][FX taps][FY taps]
    constexpr bool kHasMid = (KX != AX_ID);
    float* tin = smem;
    float* tmid = kHasMid ? smem + p.a_size : tin;
    const int mid_size = kHasMid ? p.pb * in_extent<KY, SY, FY>(p.toh) * p.p_mid : 0;
    float* s_fx = smem + p.a_size + mid_size;
    float* s_fy = s_fx + FX;

    // CTA -> (first plane, tile). With pb > 1 the CTA owns pb whole planes (tiles_x == tiles_y == 1).
    // (all 32-bit: the host bounds the grid by 2^31 - 1, so plane indices fit)
    const unsigned tiles = (unsigned)(p.tiles_x * p.tiles_y);
    const unsigned plane0 = (p.pb > 1) ? blockIdx.x * (unsigned)p.pb : (tiles > 1 ? blockIdx.x / tiles : blockIdx.x);
    const int tile = (p.pb > 1 || tiles == 1) ? 0 : (int)(blockIdx.x - plane0 * tiles);
    const int npl = (p.pb > 1) ? (int)min((int64_t)p.pb, p.planes - (int64_t)plane0) : 1;
    const int ty = (p.tiles_x > 1) ? tile / p.tiles_x : tile, tx = tile - ty * p.tiles_x;
    const int ox0 = tx * p.tow, oy0 = ty * p.toh;
    const int tow_e = min(p.tow, p.ow - ox0), toh_e = min(p.toh, p.oh - oy0);
    // plane -> memory offset: pb > 1 requires stride[0] == C * stride[1] (checked on the host)
    const unsigned pn = plane0 / (unsigned)p.c, pc = plane0 - pn * (unsigned)p.c;
    const int64_t xoff0 = (p.pb > 1) ? (int64_t)plane0 * p.xs[1] : (int64_t)pn * p.xs[0] + (int64_t)pc * p.xs[1];
    const int64_t yoff0 = (p.pb > 1) ? (int64_t)plane0 * p.ys[1] : (int64_t)pn * p.ys[0] + (int64_t)pc * p.ys[1];

    // taps oriented for correlation; the gain is folded into the taps of the y pass (or applied on store when there is none)
    if (KX != AX_ID) for (int i = threadIdx.x; i < FX; i += kThreads) s_fx[i] = p.flip ? p.fx[i * p.fsx] : p.fx[(FX - 1 - i) * p.fsx];
    if (KY != AX_ID) for (int i = threadIdx.x; i < FY; i += kThreads) s_fy[i] = p.gain * (p.flip ? p.fy[i * p.fsy] : p.fy[(FY - 1 - i) * p.fsy]);

    // per-axis geometry: first input sample of the tile, how many to load, phase offsets
    int in_x0, in_w, nqx = 0, dxo = 0;
    if (KX == AX_UP) {
        in_x0 = floordiv(ox0 - p.padx0, SX);
        dxo = (ox0 - p.padx0) - in_x0 * SX;
        nqx = (tow_e + dxo + SX - 1) / SX;
        in_w = fir::round_up(nqx, kR) + FX / SX;
    } else if (KX == AX_DOWN) {
        in_x0 = ox0 * SX - p.padx0;
        in_w = (tow_e - 1) * SX + FX;
    } else {
        in_x0 = ox0 - p.padx0;
        in_w = tow_e;
    }
    int in_y0, in_h, nqy = 0, dyo = 0;
    if (KY == AX_UP) {
        in_y0 = floordiv(oy0 - p.pady0, SY);
        dyo = (oy0 - p.pady0) - in_y0 * SY;
        nqy = (toh_e + dyo + SY - 1) / SY;
        in_h = fir::round_up(nqy, kR) + FY / SY;
    } else if (KY == AX_DOWN) {
        in_y0 = oy0 * SY - p.pady0;
        in_h = (toh_e - 1) * SY + FY;
    } else {
        in_y0 = oy0 - p.pady0;
        in_h = toh_e;
    }

    // ---- input tile(s), zero outside the image
    if (p.flat) {
        // Whole planes, contiguous in memory: zero the tile, then stream the planes with 128-bit loads
        // (4 vectors in flight per thread) and scatter the elements that fall inside the tile.
        constexpr int V = VecOf<T>::N;
        const int tile_floats = npl * in_h * p.p_in;
        for (int i = threadIdx.x; i < tile_floats; i += kThreads) tin[i] = 0.f;
        __syncthreads();
        const T* xp = (const T*)p.x + xoff0;
        const int plane_elems = p.ih * p.iw;
        const int nvec = npl * plane_elems / V;
        const fir::FastDiv by_plane = p.by_plane_elems, by_w = p.by_iw;
        const bool inside = p.flat == 2;
        constexpr int kBatch = 4;
        for (int base = threadIdx.x; base < nvec; base += kThreads * kBatch) {
            Pack<T> v[kBatch];
#pragma unroll
            for (int j = 0; j < kBatch; j++) {
                const int vi = base + j * kThreads;
                if (vi < nvec) v[j] = load_pack(xp + (int64_t)vi * V);
            }
#pragma unroll
            for (int j = 0; j < kBatch; j++) {
                const int vi = base + j * kThreads;
                if (vi < nvec) {
                    const int e = vi * V;
                    const int pl = by_plane.div(e);
                    const int rem = e - pl * plane_elems;
                    const int gy = by_w.div(rem);
                    const int gx = rem - gy * p.iw;
                    const int iy = gy - in_y0, ix = gx - in_x0;
                    float* dst = tin + (pl * in_h + iy) * p.p_in + ix;
                    if (inside) {
#pragma unroll
                        for (int k = 0; k < V; k++) dst[k] = to_acc(v[j].v[k]);
                    } else if (iy >= 0 && iy < in_h) {
#pragma unroll
                        for (int k = 0; k < V; k++)
                            if (ix + k >= 0 && ix + k < in_w) dst[k] = to_acc(v[j].v[k]);
                    }
                }
            }
        }
    } else {
        // general case: one warp per row, lanes along the row
        const T* xp = (const T*)p.x + xoff0;
        const int rows = npl * in_h;
        const fir::FastDiv by_h(in_h);
        const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
        for (int r = warp; r < rows; r += kThreads / 32) {
            const int pl = npl > 1 ? by_h.div(r) : 0;
            const int gy = in_y0 + (r - pl * in_h);
            const bool rowok = gy >= 0 && gy < p.ih;
            const T* xrow = xp + (int64_t)pl * p.xs[1] + (int64_t)gy * p.xs[2];
            for (int ix = lane; ix < in_w; ix += 32) {
                const int gx = in_x0 + ix;
                float v = 0.f;
                if (rowok && gx >= 0 && gx < p.iw) v = to_acc(xrow[(int64_t)gx * p.xs[3]]);
                tin[r * p.p_in + ix] = v;
            }
        }
    }
    __syncthreads();

    // ---- x pass
    // Packed (two outputs per FMA) passes; 24-tap down-sampling keeps the scalar form (register budget).
    int pmid = p.p_in;
    const int xshift = 0;
    if constexpr (KX == AX_UP) {
        fir::up_x2<SX, FX, kR, kThreads>(tin, p.p_in, tmid + xshift, p.p_mid, npl * in_h, nqx, s_fx);
        pmid = p.p_mid;
        __syncthreads();
    } else if constexpr (KX == AX_DOWN) {
        if constexpr (FX <= 12) fir::down_x2<SX, FX, kR, kThreads>(tin, p.p_in, 0, tmid, p.p_mid, npl * in_h, tow_e, s_fx);
        else                    fir::down_x<SX, FX, kR, kThreads>(tin, p.p_in, 0, tmid, p.p_mid, npl * in_h, tow_e, s_fx);
        pmid = p.p_mid;
        __syncthreads();
    }

    // ---- y pass -> global. The store address of a thread item is formed once (64-bit), results then only
    // add a 32-bit row offset (the host guarantees that a plane spans < 2^31 elements).
    // yp is CTA-uniform; every result adds an unsigned 32-bit element offset (the host guarantees that the
    // outputs of one CTA span < 2^31 elements), so no per-result 64-bit address arithmetic is left.
    T* yp = (T*)p.y + yoff0 + (int64_t)oy0 * p.ys[2] + (int64_t)ox0 * p.ys[3];
    const float gain = p.gain;
    const float* src = tmid + dxo + xshift;
    const int ys1 = (int)p.ys[1], ys2 = (int)p.ys[2], ys3 = (int)p.ys[3];
    if constexpr (KY == AX_UP) {
        up_y2_store<T, SY, FY, kR, kThreads>(src, pmid, tow_e, nqy, s_fy, yp, ys1, ys2, ys3, dyo, toh_e, npl, in_h);
    } else if constexpr (KY == AX_DOWN) {
        if constexpr (FY <= 12) {
            down_y2_store<T, SY, FY, kR, kThreads>(src, pmid, tow_e, toh_e, s_fy, yp, ys1, ys2, ys3, npl, in_h);
        } else {
            const unsigned uys1 = (unsigned)ys1, uys2 = (unsigned)ys2, uys3 = (unsigned)ys3;
            fir::down_y<SY, FY, kR, kThreads>(src, pmid, 0, tow_e, toh_e, s_fy,
                fir::make_emitter([&](int pl, int col) { return (unsigned)pl * uys1 + (unsigned)col * uys3; },
                                  [&](unsigned off, int o, float acc) { yp[off + (unsigned)o * uys2] = from_acc<T>(acc); }), npl, in_h);
        }
    } else {
        const int per = toh_e * tow_e;
        const fir::FastDiv by_w(tow_e), by_per(per);
        for (int idx = threadIdx.x; idx < npl * per; idx += kThreads) {
            const int pl = npl > 1 ? by_per.div(idx) : 0;
            const int rem = idx - pl * per;
            const int o = by_w.div(rem), col = rem - o * tow_e;
            yp[(unsigned)(pl * ys1 + o * ys2 + col * ys3)] = from_acc<T>(src[(pl * in_h + o) * pmid + col] * gain);
        }
    }
}

// whole rows up to 256 pixels, else the widest tile <= 128 that wastes the fewest lanes of the 32-wide column chunks
int pick_tow(int ow)
{
    if (ow <= 256) return ow;
    int best = 64, best_waste = INT32_MAX;
    for (int cand = 128; cand >= 64; cand -= 32) {
        const int tiles = (ow + cand - 1) / cand;
        const int last = ow - (tiles - 1) * cand;
        const int waste = tiles * cand - ow + (fir::round_up(last, 32) - last);
        if (waste < best_waste) { best_waste = waste; best = cand; }
    }
    return best;
}

template <class T, int KX, int SX, int FX, int KY, int SY, int FY>
int launch_tiled(TiledParams& p, cudaStream_t s)
{
    static const int kTargetOutputs = [] {      // outputs per CTA the tile/plane batching aims for
        const char* e = getenv("LVG_UPFIRDN_TARGET");
        const int v = e ? atoi(e) : 0;
        return v >= 1024 ? v : 16384;
    }();
    constexpr size_t kSmemBudget = 56 * 1024;   // keeps 4 CTAs resident per SM
    p.tow = pick_tow(p.ow);
    int toh = kTargetOutputs / (p.tow > 0 ? p.tow : 1);
    toh = fir::round_up(toh < 4 ? 4 : toh, 4);
    if (toh > p.oh) toh = p.oh;
    p.pb = 1;
    auto smem_for = [&](int toh_, int pb_) {
        const int in_w = in_extent<KX, SX, FX>(p.tow), in_h = in_extent<KY, SY, FY>(toh_);
        p.p_in = fir::odd_pitch(in_w);
        p.p_mid = fir::odd_pitch(mid_extent<KX, SX, FX>(p.tow) + (KX == AX_UP ? SX : 0));
        p.a_size = pb_ * in_h * p.p_in;
        const int mid = (KX == AX_ID) ? 0 : pb_ * in_h * p.p_mid;
        return (size_t)(p.a_size + mid + FX + FY) * sizeof(float);
    };
    // the whole plane fits: one tile per plane (vector loader, no halo re-reads, plane batching below)
    if (p.tow == p.ow && smem_for(p.oh, 1) <= kSmemBudget) toh = p.oh;
    size_t smem = smem_for(toh, 1);       // (smem_for also records the pitches / tile sizes in p: call it last for the choice made)
    while (smem > kSmemBudget && toh > 4) {
        toh = fir::round_up(toh / 2, 4);
        smem = smem_for(toh, 1);
    }
    if (smem > 200 * 1024) return LVG_UNSUPPORTED;
    p.toh = toh;
    p.tiles_x = (p.ow + p.tow - 1) / p.tow;
    p.tiles_y = (p.oh + p.toh - 1) / p.toh;
    // small planes: several whole planes per CTA (needs planes to be equally spaced in memory)
    const bool uniform = (p.xs[0] == (int64_t)p.c * p.xs[1]) && (p.ys[0] == (int64_t)p.c * p.ys[1]);
    if (p.tiles_x == 1 && p.tiles_y == 1 && uniform && p.planes > 1) {
        int pb = kTargetOutputs / (p.ow * p.oh);
        if (pb > 64) pb = 64;
        if ((int64_t)pb > p.planes) pb = (int)p.planes;
        while (pb > 1 && smem_for(p.toh, pb) > kSmemBudget) pb--;
        if (pb < 1) pb = 1;
        p.pb = pb;
        smem = smem_for(p.toh, p.pb);
    }
    // vector loader: whole contiguous planes, rows a multiple of the 16-byte vector, aligned base
    constexpr int V = VecOf<T>::N;
    p.flat = (p.tiles_x == 1 && p.tiles_y == 1 && p.xs[3] == 1 && p.xs[2] == p.iw && p.xs[1] == (int64_t)p.ih * p.iw &&
              (p.pb == 1 || uniform) && p.iw % V == 0 && p.xs[0] % V == 0 && aligned16(p.x) && (int64_t)p.pb * p.ih * p.iw < (1 << 24)) ? 1 : 0;
    if (p.flat) {
        p.by_plane_elems = fir::FastDiv(p.ih * p.iw);
        p.by_iw = fir::FastDiv(p.iw);
        // does the (single) tile contain every input sample? then the scatter needs no bounds checks
        const int in_x0 = KX == AX_UP ? floordiv(-p.padx0, SX) : -p.padx0;
        const int in_y0 = KY == AX_UP ? floordiv(-p.pady0, SY) : -p.pady0;
        const int in_w = KX == AX_UP ? fir::round_up((p.ow + (-p.padx0 - in_x0 * SX) + SX - 1) / SX, kR) + FX / SX
                       : KX == AX_DOWN ? (p.ow - 1) * SX + FX : p.ow;
        const int in_h = KY == AX_UP ? fir::round_up((p.oh + (-p.pady0 - in_y0 * SY) + SY - 1) / SY, kR) + FY / SY
                       : KY == AX_DOWN ? (p.oh - 1) * SY + FY : p.oh;
        if (in_x0 <= 0 && in_y0 <= 0 && p.iw - in_x0 <= in_w && p.ih - in_y0 <= in_h) p.flat = 2;
    }
    // 32-bit output offsets inside one CTA's share of y
    {
        auto mag = [](int64_t v) { return v < 0 ? -v : v; };
        for (int i = 0; i < 4; i++) if (p.ys[i] < 0) return LVG_UNSUPPORTED;
        const int64_t span = (int64_t)(p.pb - 1) * mag(p.ys[1]) + (int64_t)(p.toh - 1) * mag(p.ys[2]) + (int64_t)(p.tow - 1) * mag(p.ys[3]);
        if (span >= (1ll << 31) || p.ys[1] >= (1ll << 32) || p.ys[2] >= (1ll << 32) || p.ys[3] >= (1ll << 32)) return LVG_UNSUPPORTED;
    }
    const int64_t blocks = p.pb > 1 ? (p.planes + p.pb - 1) / p.pb : p.planes * p.tiles_x * p.tiles_y;
    if (blocks > INT32_MAX) return LVG_UNSUPPORTED;
    // (one CTA per work item: a persistent grid prefetching the next item's vectors costs live registers and resident CTAs)
    auto k = upfirdn2d_tiled_kernel<T, KX, SX, FX, KY, SY, FY>;
    if (smem > 48 * 1024) LVG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<(unsigned)blocks, kThreads, smem, s>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

struct Axis { int kind, s, f; };

Axis classify(bool has_filter, int up, int down, int taps)
{
    if (!has_filter && up == 1 && down == 1) return {AX_ID, 1, 1};
    if (!has_filter) return {-1, 0, 0};
    if (up > 1 && down == 1 && taps % up == 0) return {AX_UP, up, taps};
    if (up == 1) return {AX_DOWN, down, taps};
    return {-1, 0, 0};
}

#define LVG_TILED_CASE(kx, sx, fx_, ky, sy, fy_)                                                        \
    if (ax.kind == kx && ax.s == sx && ax.f == fx_ && ay.kind == ky && ay.s == sy && ay.f == fy_)       \
        return launch_tiled<T, kx, sx, fx_, ky, sy, fy_>(p, s);

template <class T>
int dispatch(const Axis& ax, const Axis& ay, TiledParams& p, cudaStream_t s)
{
    // the resampling signatures of the LongVideoGAN networks and their adjoints (SURVEY.md Appendix A)
    LVG_TILED_CASE(AX_UP, 2, 4, AX_UP, 2, 4)          // U3  bilinear 2x spatial up-sampling
    LVG_TILED_CASE(AX_DOWN, 2, 4, AX_DOWN, 2, 4)      // U4  2x spatial down-sampling (and adjoint of U3)
    LVG_TILED_CASE(AX_ID, 1, 1, AX_UP, 2, 4)          // U2  temporal linear up-sampling
    LVG_TILED_CASE(AX_ID, 1, 1, AX_DOWN, 2, 4)        // U5  temporal down-sampling
    LVG_TILED_CASE(AX_ID, 1, 1, AX_DOWN, 2, 12)       // U1  temporal Kaiser down-sampling
    LVG_TILED_CASE(AX_ID, 1, 1, AX_UP, 2, 12)         //     adjoint of U1
    LVG_TILED_CASE(AX_DOWN, 2, 12, AX_ID, 1, 1)       // U1  on [N, C, L, 1] tensors (transposed view: filter along x)
    LVG_TILED_CASE(AX_UP, 2, 12, AX_ID, 1, 1)         //     and its adjoint
    LVG_TILED_CASE(AX_DOWN, 4, 24, AX_DOWN, 4, 24)    // U6  Kaiser down 4
    LVG_TILED_CASE(AX_DOWN, 2, 12, AX_DOWN, 2, 12)    // U6 / U9 down 2, 12 taps
    LVG_TILED_CASE(AX_UP, 2, 12, AX_UP, 2, 12)        // U6 / U9 up 2, 12 taps
    LVG_TILED_CASE(AX_UP, 4, 24, AX_UP, 4, 24)        // U6  Kaiser up 4
    LVG_TILED_CASE(AX_UP, 4, 8, AX_UP, 4, 8)          // U7  4x up-sampling of the low-res frames
    LVG_TILED_CASE(AX_DOWN, 4, 8, AX_DOWN, 4, 8)      //     adjoint of U7
    LVG_TILED_CASE(AX_DOWN, 1, 4, AX_DOWN, 1, 4)      // U8  4x4 blur before a strided convolution
    return LVG_UNSUPPORTED;
}

}  // namespace

// shared by lvg_upfirdn2d (rank-1-in-one-axis filters) and lvg_upfirdn2d_sep
int upfirdn2d_tiled(const void* x, const float* fx, int64_t fsx, const float* fy, int64_t fsy, void* y, int dtype,
                    const int64_t* xsh, const int64_t* xst, const int64_t* ysh, const int64_t* yst,
                    int fw, int fh, int upx, int upy, int downx, int downy, int padx0, int pady0,
                    int flip, float gain, cudaStream_t s)
{
    if (dtype != LVG_F32 && dtype != LVG_F16) return LVG_UNSUPPORTED;
    // the 2x / 4-tap signatures of the low-res networks stream through registers (upfirdn2d_stream.cu)
    {
        const int rc = upfirdn2d_stream(x, fx, fsx, fy, fsy, y, dtype, xsh, xst, ysh, yst, fw, fh, upx, upy, downx, downy, padx0, pady0, flip, gain, s);
        if (rc != LVG_UNSUPPORTED) return rc;
    }
    const Axis ax = classify(fx != nullptr, upx, downx, fw), ay = classify(fy != nullptr, upy, downy, fh);
    if (ax.kind < 0 || ay.kind < 0) return LVG_UNSUPPORTED;
    TiledParams p;
    p.x = x; p.fx = fx; p.fy = fy; p.y = y;
    for (int i = 0; i < 4; i++) { p.xs[i] = xst[i]; p.ys[i] = yst[i]; }
    p.fsx = fsx; p.fsy = fsy;
    p.n = (int)xsh[0]; p.c = (int)xsh[1]; p.ih = (int)xsh[2]; p.iw = (int)xsh[3];
    p.oh = (int)ysh[2]; p.ow = (int)ysh[3];
    p.planes = (int64_t)p.n * p.c;
    p.padx0 = padx0; p.pady0 = pady0; p.flip = flip ? 1 : 0; p.gain = gain;
    return dtype == LVG_F32 ? dispatch<float>(ax, ay, p, s) : dispatch<__half>(ax, ay, p, s);
}

}  // namespace lvg

using namespace lvg;

extern "C" int lvg_upfirdn2d_sep(const void* x, const float* fx, const float* fy, void* y,
                                 int dtype, const int64_t x_shape[4], const int64_t x_stride[4],
                                 const int64_t y_shape[4], const int64_t y_stride[4],
                                 int fw, int fh, int upx, int upy, int downx, int downy,
                                 int padx0, int pady0, int flip, float gain, void* stream)
{
    int rc = upfirdn2d_check(x, y, dtype, x_shape, y_shape, fw, fh, upx, upy, downx, downy);
    if (rc) return rc;
    LVG_REQUIRE((fx != nullptr) || fw == 1, "upfirdn2d_sep: fx == NULL requires fw == 1");
    LVG_REQUIRE((fy != nullptr) || fh == 1, "upfirdn2d_sep: fy == NULL requires fh == 1");
    rc = upfirdn2d_tiled(x, fx, 1, fy, 1, y, dtype, x_shape, x_stride, y_shape, y_stride, fw, fh, upx, upy,
                         downx, downy, padx0, pady0, flip, gain, (cudaStream_t)stream);
    if (rc == LVG_UNSUPPORTED) set_error("upfirdn2d_sep: no tiled kernel for this configuration");
    return rc;
}
