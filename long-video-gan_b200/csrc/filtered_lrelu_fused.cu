// Fused filtered leaky ReLU: bias -> up-FIR -> gain*lrelu*clamp (+ 2-bit signs) -> down-FIR
// in ONE kernel; the up-sampled intermediate (4x / 16x the input) never leaves shared memory.
//
// Semantics follow the reference kernel (torch_utils/ops/filtered_lrelu.cu:139-1099) and
// _filtered_lrelu_ref (filtered_lrelu.py:121-153):
//   t[U]   = up^2 * sum_s gu[s] * z[U + s - pad0],  z = zero-stuffed (x + b), zero outside the image
//   v      = t * gain;  write/plain: v < 0 -> v *= slope (code 1); |v| > clamp -> +-clamp (code 2)
//            read: code = signs[U + sx, V + sy]; bit0 -> v *= slope; bit1 -> v = 0; outside the tensor: unchanged
//   y[o]   = sum_t gd[t] * v[o*down + t]
// for separable filters (the only kind the networks use), per axis.
//
// One CTA = one TOW x TOH output tile of one (n, c) plane, five stages through two shared-memory
// buffers (A: input tile, then the activated up-sampled tile; B: x-up-sampled rows, then
// x-down-sampled rows). All passes are the register-blocked polyphase routines of fir_passes.cuh.
// Filters arrive as device pointers and are staged per CTA in shared memory -- no global
// __constant__ state (the reference's c_fbuf, filtered_lrelu.cu:78), so the op is stream-safe.
// Sign bytes are packed from a per-sample code tile in shared memory; every CTA owns a
// byte-aligned slab of the sign tensor, so no two CTAs touch the same byte.

#include "common.cuh"
#include "fir_passes.cuh"
#include "filtered_lrelu_v3.cuh"
#include <stdlib.h>

namespace lvg {
namespace flv3 {
template <class T> int launch(int cfg, FlParams& p, int mode, cudaStream_t s);     // filtered_lrelu_v3.cu
}
namespace {
using flv3::FlParams;

enum { SIGN_NONE = 0, SIGN_WRITE = 1, SIGN_READ = 2 };


constexpr int kThreads = 256;
constexpr int kR = 4;       // outputs (down passes) / input groups (up passes) per thread

template <int UP, int FU, int DOWN, int FD, int TOW, int TOH>
struct Geom {
    static constexpr int KU = FU / UP;
    static constexpr int TUW = (TOW - 1) * DOWN + FD;                 // up-sampled samples the tile consumes
    static constexpr int TUH = (TOH - 1) * DOWN + FD;
    static constexpr int NQX = (TUW + UP - 1 + UP - 1) / UP;          // phase-aligned groups incl. alignment slack
    static constexpr int NQY = (TUH + UP - 1 + UP - 1) / UP;
    static constexpr int NQXR = fir::round_up(NQX, kR);
    static constexpr int NQYR = fir::round_up(NQY, kR);
    static constexpr int TUWA = NQXR * UP;                            // computed (aligned) up-sampled extent
    static constexpr int TUHA = NQYR * UP;
    static constexpr int TIW = NQXR + KU;                             // input tile incl. filter support
    static constexpr int TIH = NQYR + KU;
    static constexpr int P_IN = fir::odd_pitch(TIW);
    static constexpr int P_UX = fir::odd_pitch(TUWA);
    static constexpr int P_UXY = fir::odd_pitch(fir::round_up(TUWA + DOWN * kR, 2));   // slack for the down-x overrun
    static constexpr int TOWR = fir::round_up(TOW, kR);
    static constexpr int TOHR = fir::round_up(TOH, kR);
    static constexpr int P_DX = fir::odd_pitch(TOWR);
    static constexpr int UXY_ROWS = TUHA + DOWN * kR;                 // slack rows for the down-y overrun
    static constexpr int A_SIZE = (TIH * P_IN > UXY_ROWS * P_UXY) ? TIH * P_IN : UXY_ROWS * P_UXY;
    static constexpr int B_SIZE = (TIH * P_UX > UXY_ROWS * P_DX) ? TIH * P_UX : UXY_ROWS * P_DX;
    static constexpr int CODE_BYTES = fir::round_up(TUHA * TUWA, 16);
    static constexpr int SIGN_PITCH = TUWA / 4 + 2;                   // sign bytes per staged row (read mode)
    static constexpr int SIGN_BYTES = fir::round_up(TUHA * SIGN_PITCH, 16);
    static constexpr size_t smem_bytes(int mode) {
        return (size_t)(A_SIZE + B_SIZE + FU + FD) * sizeof(float) + (mode == SIGN_WRITE ? CODE_BYTES : mode == SIGN_READ ? SIGN_BYTES : 0);
    }
};

template <class T, int UP, int FU, int DOWN, int FD, int TOW, int TOH, int MODE>
__global__ void __launch_bounds__(kThreads, (TOH <= 24 ? 3 : 2)) filtered_lrelu_kernel(FlParams p)
{
    typedef Geom<UP, FU, DOWN, FD, TOW, TOH> G;
    extern __shared__ __align__(16) float smem[];
    float* bufA = smem;
    float* bufB = bufA + G::A_SIZE;
    float* s_fu = bufB + G::B_SIZE;
    float* s_fd = s_fu + FU;
    uint8_t* s_code = reinterpret_cast<uint8_t*>(s_fd + FD);

    // (32-bit unsigned index arithmetic: the host bounds the grid by 2^31 - 1 CTAs)
    const unsigned tiles = (unsigned)(p.tiles_x * p.tiles_y);
    const unsigned plane = blockIdx.x / tiles;
    const unsigned tile = blockIdx.x - plane * tiles;
    const int ty = (int)(tile / (unsigned)p.tiles_x), tx = (int)tile - ty * p.tiles_x;
    const int ox0 = tx * TOW, oy0 = ty * TOH;
    const int nn = (int)(plane / (unsigned)p.c);
    const int cc = (int)(plane - (unsigned)nn * (unsigned)p.c);

    // The factor up^2 * gain that precedes the leaky ReLU is positive, so it is folded into the up-sampling
    // taps (its square root into each of the two passes) instead of costing a multiply per up-sampled sample.
    {
        const float tap_scale = sqrtf((float)(UP * UP) * p.gain);
        for (int i = threadIdx.x; i < FU; i += kThreads) s_fu[i] = (p.flip ? p.fu[i] : p.fu[FU - 1 - i]) * tap_scale;
    }
    fir::load_taps(s_fd, p.fd, FD, p.flip != 0);

    // geometry of this tile: U0 = first consumed up-sampled sample; the phase-aligned origin is
    // Ua = U0 - dxo with (Ua - pad0) a multiple of UP; m0 = first input sample of group 0
    const int U0 = ox0 * DOWN, V0 = oy0 * DOWN;
    const int m0x = floordiv(U0 - p.px0, UP), m0y = floordiv(V0 - p.py0, UP);
    const int dxo = (U0 - p.px0) - m0x * UP, dyo = (V0 - p.py0) - m0y * UP;
    const int tow_e = min(TOW, p.ow - ox0), toh_e = min(TOH, p.oh - oy0);
    const int tuw_e = (tow_e - 1) * DOWN + FD, tuh_e = (toh_e - 1) * DOWN + FD;
    const int nqx_e = (tuw_e + dxo + UP - 1) / UP, nqy_e = (tuh_e + dyo + UP - 1) / UP;
    const int tiw_e = fir::round_up(nqx_e, kR) + G::KU, tih_e = fir::round_up(nqy_e, kR) + G::KU;

    // ---- stage 0 (read mode): this tile's slab of the sign tensor -> shared memory with coalesced byte loads, issued first
    // so that their latency hides behind stages 1-2 (per-sample global byte loads in stage 3 cost 40 % of the kernel:
    // long-scoreboard stalls). Bytes outside the tensor read as 0 = "unchanged", the operator's rule for such samples.
    const int sgn_bx0 = (U0 - dxo + p.sx) >> 2;            // first staged byte column (floor division also for negatives)
    if (MODE == SIGN_READ) {
        const uint8_t* sgn = p.si + plane * (int64_t)p.s_h * p.s_wb;
        const int gy0 = V0 - dyo + p.sy;
        for (int i = threadIdx.x; i < G::TUHA * G::SIGN_PITCH; i += kThreads) {
            const int row = i / G::SIGN_PITCH, bb = i - row * G::SIGN_PITCH;
            const int gy = gy0 + row, gb = sgn_bx0 + bb;
            uint8_t v = 0;
            if ((unsigned)gy < (unsigned)p.s_h && (unsigned)gb < (unsigned)p.s_wb) v = __ldg(sgn + (int64_t)gy * p.s_wb + gb);
            s_code[i] = v;
        }
    }

    // ---- stage 1: input tile (+ bias inside the image, zero outside) -> A
    // One warp per tile row, lanes along the row; the loop nest has compile-time trip counts and is fully
    // unrolled, so all of a thread's global loads are in flight before the first shared-memory store, and the
    // per-element work is a predicated load, a convert, the bias add and the store (row / column validity and
    // the row pointer are computed once per row / per lane-column).
    {
        const T* xp = (const T*)p.x + (int64_t)nn * p.xs[0] + (int64_t)cc * p.xs[1];
        const float bias = to_acc(((const T*)p.b)[cc]);
        constexpr int kWarps = kThreads / 32;
        constexpr int kRowIters = (G::TIH + kWarps - 1) / kWarps;
        constexpr int kColIters = (G::TIW + 31) / 32;
        const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
        // offsets inside one (n, c) plane fit 32 bits (checked on the host): one IMAD per row, one add per element
        const int xs2 = (int)p.xs[2], xs3 = (int)p.xs[3];
        bool colok[kColIters];
        int coloff[kColIters];
#pragma unroll
        for (int cj = 0; cj < kColIters; cj++) {
            const int ix = lane + 32 * cj, gx = m0x + ix;
            colok[cj] = ix < tiw_e && gx >= 0 && gx < p.iw;
            coloff[cj] = gx * xs3;
        }
        float v[kRowIters][kColIters];
#pragma unroll
        for (int ri = 0; ri < kRowIters; ri++) {
            const int iy = warp + kWarps * ri, gy = m0y + iy;
            const bool rowok = iy < tih_e && gy >= 0 && gy < p.ih;
            const int rowoff = gy * xs2;
#pragma unroll
            for (int cj = 0; cj < kColIters; cj++) {
                v[ri][cj] = 0.f;
                if (rowok && colok[cj]) v[ri][cj] = to_acc(xp[rowoff + coloff[cj]]) + bias;
            }
        }
#pragma unroll
        for (int ri = 0; ri < kRowIters; ri++) {
            const int iy = warp + kWarps * ri;
#pragma unroll
            for (int cj = 0; cj < kColIters; cj++) {
                const int ix = lane + 32 * cj;
                if (iy < G::TIH && ix < G::TIW) bufA[iy * G::P_IN + ix] = v[ri][cj];
            }
        }
    }
    __syncthreads();

    // ---- stage 2: up-sample along x: A [tih][tiw] -> B [tih][TUWA]   (packed FMA: two rows per thread)
    fir::up_x2<UP, FU, kR, kThreads>(bufA, G::P_IN, bufB, G::P_UX, tih_e, nqx_e, s_fu);
    __syncthreads();

    // ---- stage 3: up-sample along y, scale, activation, signs: B -> A [TUHA][TUWA]   (two columns per thread)
    {
        const float slope = p.slope, clamp = p.clamp;
        const bool shrink = slope <= 1.f;                  // lrelu(v) = max(v, v*slope) for slope <= 1, min(...) otherwise
        const int Uax = U0 - dxo, Vay = V0 - dyo;          // global up-sampled coords of aligned sample (0, 0)
        const int cols = nqx_e * UP;
        const int qx0 = Uax + p.sx;
        (void)Vay;
        auto activate = [&](float v, int row, int col, unsigned& code) {
            if (MODE == SIGN_READ) {
                const int qx = qx0 + col;
                const unsigned s = (unsigned)s_code[row * G::SIGN_PITCH + ((qx >> 2) - sgn_bx0)] >> ((qx & 3) << 1);
                v = (s & 1u) ? v * slope : v;
                v = (s & 2u) ? 0.f : v;
            } else if (MODE == SIGN_WRITE) {
                // branch-free: selects only (the sign code is 2 if clamped, else 1 if negative)
                const bool neg = v < 0.f;
                v = neg ? v * slope : v;
                const bool sat = fabsf(v) > clamp;
                v = fminf(fmaxf(v, -clamp), clamp);
                code = sat ? 2u : (neg ? 1u : 0u);
            } else {
                const float vs = v * slope;
                v = shrink ? fmaxf(v, vs) : fminf(v, vs);
                v = fminf(fmaxf(v, -clamp), clamp);
            }
            return v;
        };
        fir::up_y2<UP, FU, kR, kThreads>(bufB, G::P_UX, cols, nqy_e, s_fu,
            [&](int, int row, int col, float acc) {
                unsigned code = 0;
                const float v = activate(acc, row, col, code);
                if (MODE == SIGN_WRITE) s_code[row * G::TUWA + col] = (uint8_t)code;
                bufA[row * G::P_UXY + col] = v;
            });
    }
    __syncthreads();

    // ---- stage 3b: pack and store this CTA's slab of the sign tensor
    if (MODE == SIGN_WRITE) {
        const bool lastx = (tx == p.tiles_x - 1), lasty = (ty == p.tiles_y - 1);
        const int b0 = U0 >> 2;                                              // TOW*DOWN is a multiple of 4
        const int b1 = lastx ? p.s_wb : min(p.s_wb, (U0 + TOW * DOWN) >> 2);
        const int r0 = V0;
        const int r1 = lasty ? p.s_h : min(p.s_h, V0 + TOH * DOWN);
        const int nb = b1 - b0, nr = r1 - r0;
        uint8_t* dst = p.so + plane * (int64_t)p.s_h * p.s_wb;
        const int cols = nqx_e * UP, rows = nqy_e * UP;
        for (int i = threadIdx.x; i < nb * nr; i += kThreads) {
            const int rr = i / nb, bb = i - rr * nb;
            const int row = rr + dyo;                                        // local aligned row of global row r0 + rr
            unsigned byte = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int U = (b0 + bb) * 4 + k;
                const int col = U - (U0 - dxo);
                if (U < p.sw_active && col < cols && row < rows)
                    byte |= (unsigned)s_code[row * G::TUWA + col] << (2 * k);
            }
            dst[(int64_t)(r0 + rr) * p.s_wb + b0 + bb] = (uint8_t)byte;
        }
    }

    // ---- stage 4: down-sample along x: A [tuh][.] (from column dxo, rows from dyo) -> B [tuh][TOW]
    // ---- stage 5: down-sample along y and store. 24-tap filters keep the one-output-per-FMA form (registers).
    T* yp = (T*)p.y + (int64_t)nn * p.ys[0] + (int64_t)cc * p.ys[1] + (int64_t)oy0 * p.ys[2] + (int64_t)ox0 * p.ys[3];
    const int64_t ys2 = p.ys[2], ys3 = p.ys[3];
    const int ys2_32 = (int)p.ys[2];          // a plane spans < 2^31 elements (checked on the host)
    if constexpr (FD <= 12) {
        fir::down_x2<DOWN, FD, kR, kThreads>(bufA + dyo * G::P_UXY, G::P_UXY, dxo, bufB, G::P_DX, tuh_e, tow_e, s_fd);
        __syncthreads();
        fir::down_y2<DOWN, FD, kR, kThreads>(bufB, G::P_DX, 0, tow_e, toh_e, s_fd,
            fir::make_emitter([&](int, int col) { return yp + col * ys3; },
                              [&](T* base, int o, float acc) { base[o * ys2_32] = from_acc<T>(acc); }));
    } else {
        fir::down_x<DOWN, FD, kR, kThreads>(bufA + dyo * G::P_UXY, G::P_UXY, dxo, bufB, G::P_DX, tuh_e, tow_e, s_fd);
        __syncthreads();
        fir::down_y<DOWN, FD, kR, kThreads>(bufB, G::P_DX, 0, tow_e, toh_e, s_fd,
            [&](int, int o, int col, float acc) { yp[o * ys2 + col * ys3] = from_acc<T>(acc); });
    }
}

// up = down = 1 with 1x1 filters (the ToRGB layer): an element-wise op; one thread = one sign byte.
template <class T, int MODE>
__global__ void __launch_bounds__(256) filtered_lrelu_1x1_kernel(FlParams p, int64_t total, int wq)
{
    const float fu = p.fu[0], fd = p.fd[0];
    const float scale = fu * p.gain;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int q = (int)(idx % wq);
        int64_t r = idx / wq;
        const int yy = (int)(r % p.oh);
        const int64_t plane = r / p.oh;
        const int cc = (int)(plane % p.c), nn = (int)(plane / p.c);
        const float bias = to_acc(((const T*)p.b)[cc]);
        // output pixel (ox, oy) reads input pixel (ox - px0, oy - py0)
        const T* xp = (const T*)p.x + (int64_t)nn * p.xs[0] + (int64_t)cc * p.xs[1];
        T* yp = (T*)p.y + (int64_t)nn * p.ys[0] + (int64_t)cc * p.ys[1] + (int64_t)yy * p.ys[2];
        const int iy = yy - p.py0;
        unsigned byte = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int ox = q * 4 + k;
            if (ox >= p.ow) continue;
            const int ix = ox - p.px0;
            float v = 0.f;
            if (ix >= 0 && ix < p.iw && iy >= 0 && iy < p.ih) v = to_acc(xp[(int64_t)iy * p.xs[2] + (int64_t)ix * p.xs[3]]) + bias;
            v *= scale;
            if (MODE == SIGN_READ) {
                const int qx = ox + p.sx, qy = yy + p.sy;
                if ((unsigned)qx < (unsigned)(p.s_wb * 4) && (unsigned)qy < (unsigned)p.s_h) {
                    const unsigned s = p.si[(plane * p.s_h + qy) * p.s_wb + (qx >> 2)] >> ((qx & 3) << 1);
                    if (s & 1u) v *= p.slope;
                    if (s & 2u) v = 0.f;
                }
            } else {
                unsigned code = 0;
                if (v < 0.f) { v *= p.slope; code = 1; }
                if (fabsf(v) > p.clamp) { v = v < 0.f ? -p.clamp : p.clamp; code = 2; }
                byte |= code << (2 * k);
            }
            yp[(int64_t)ox * p.ys[3]] = from_acc<T>(v * fd);
        }
        if (MODE == SIGN_WRITE && q < p.s_wb && yy < p.s_h)
            p.so[(plane * p.s_h + yy) * p.s_wb + q] = (uint8_t)byte;
    }
}

template <class T, int UP, int FU, int DOWN, int FD, int TOW, int TOH>
int launch_cfg(FlParams& p, int mode, cudaStream_t s)
{
    typedef Geom<UP, FU, DOWN, FD, TOW, TOH> G;
    static_assert((TOW * DOWN) % 4 == 0, "sign slabs must be byte aligned");
    p.tiles_x = (p.ow + TOW - 1) / TOW;
    p.tiles_y = (p.oh + TOH - 1) / TOH;
    const int64_t blocks = (int64_t)p.n * p.c * p.tiles_x * p.tiles_y;
    LVG_REQUIRE(blocks <= INT32_MAX, "filtered_lrelu: grid too large");
    const size_t smem = G::smem_bytes(mode);
    void (*k)(FlParams) = nullptr;
    if (mode == SIGN_WRITE)     k = filtered_lrelu_kernel<T, UP, FU, DOWN, FD, TOW, TOH, SIGN_WRITE>;
    else if (mode == SIGN_READ) k = filtered_lrelu_kernel<T, UP, FU, DOWN, FD, TOW, TOH, SIGN_READ>;
    else                        k = filtered_lrelu_kernel<T, UP, FU, DOWN, FD, TOW, TOH, SIGN_NONE>;
    LVG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<(unsigned)blocks, kThreads, smem, s>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

template <class T>
int launch_1x1(FlParams& p, int mode, cudaStream_t s)
{
    const int wq = max((p.ow + 3) / 4, mode == SIGN_WRITE ? p.s_wb : 0);
    const int64_t total = (int64_t)p.n * p.c * p.oh * wq;
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 8 * 16;
    if (blocks > cap) blocks = cap;
    if (mode == SIGN_WRITE)     filtered_lrelu_1x1_kernel<T, SIGN_WRITE><<<(unsigned)blocks, 256, 0, s>>>(p, total, wq);
    else if (mode == SIGN_READ) filtered_lrelu_1x1_kernel<T, SIGN_READ><<<(unsigned)blocks, 256, 0, s>>>(p, total, wq);
    else                        filtered_lrelu_1x1_kernel<T, SIGN_NONE><<<(unsigned)blocks, 256, 0, s>>>(p, total, wq);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

// configuration table: separable filters only (height 0), the four shapes of SURVEY.md Appendix A
enum Cfg { CFG_NONE = 0, CFG_1x1, CFG_U2D2, CFG_U4D2, CFG_U2D4 };

Cfg pick(int fu_w, int fu_h, int fd_w, int fd_h, int up, int down)
{
    if (up == 1 && down == 1 && fu_w == 1 && fu_h == 1 && fd_w == 1 && fd_h == 1) return CFG_1x1;
    if (fu_h != 0 || fd_h != 0) return CFG_NONE;
    if (up == 2 && fu_w == 12 && down == 2 && fd_w == 12) return CFG_U2D2;
    if (up == 4 && fu_w == 24 && down == 2 && fd_w == 12) return CFG_U4D2;
    if (up == 2 && fu_w == 12 && down == 4 && fd_w == 24) return CFG_U2D4;
    return CFG_NONE;
}

// Output tile height. 64x24 tiles fit three CTAs per SM (66 KB, <= 85 registers) against two of 64x32; the up4
// configuration has a larger halo, for which the taller tile pads fewer rows.
// An image that a single 32-row tile covers keeps the tall tile. LVG_FL_TOH=24|32 overrides (experiments).
int tile_rows(int up, int oh)
{
    static int forced = -1;
    if (forced < 0) { const char* e = getenv("LVG_FL_TOH"); forced = e ? atoi(e) : 0; }
    if (forced == 24 || forced == 32) return forced;
    (void)up;
    // fewest padded rows wins, ties go to the 24-row tile (3 CTAs per SM); LVG_FL_TOH forces one for measurements
    const int pad24 = (oh + 23) / 24 * 24, pad32 = (oh + 31) / 32 * 32;
    return pad32 < pad24 ? 32 : 24;
}

// LVG_FL_ENGINE=r2 keeps the scalar-access kernels of this file (A/B measurements); default: the vectorised kernels
bool use_v3()
{
    static int v = -1;
    if (v < 0) { const char* e = getenv("LVG_FL_ENGINE"); v = (e && e[0] == 'r' && e[1] == '2') ? 0 : 1; }
    return v == 1;
}

template <class T>
int dispatch(Cfg cfg, FlParams& p, int mode, cudaStream_t s)
{
    // the vectorised kernels serve slope <= 1 (leaky ReLU as a max) and word-aligned sign rows; anything else: the kernels below
    const bool v3_ok = p.slope <= 1.f && (mode != SIGN_READ || (p.s_wb % 4 == 0 && (reinterpret_cast<uintptr_t>(p.si) & 3) == 0));
    if (use_v3() && v3_ok && (cfg == CFG_U2D2 || cfg == CFG_U4D2 || cfg == CFG_U2D4))
        return flv3::launch<T>(cfg == CFG_U2D2 ? 1 : cfg == CFG_U4D2 ? 2 : 3, p, mode, s);
    switch (cfg) {
        case CFG_1x1:  return launch_1x1<T>(p, mode, s);
        case CFG_U2D2: { const int r = tile_rows(2, p.oh);
                         return r == 32 ? launch_cfg<T, 2, 12, 2, 12, 64, 32>(p, mode, s) : launch_cfg<T, 2, 12, 2, 12, 64, 24>(p, mode, s); }
        case CFG_U4D2: { const int r = tile_rows(4, p.oh);
                         return r == 32 ? launch_cfg<T, 4, 24, 2, 12, 64, 32>(p, mode, s) : launch_cfg<T, 4, 24, 2, 12, 64, 24>(p, mode, s); }
        case CFG_U2D4: return launch_cfg<T, 2, 12, 4, 24, 32, 16>(p, mode, s);
        default: break;
    }
    return LVG_UNSUPPORTED;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int lvg_filtered_lrelu_supported(int dtype, int fu_w, int fu_h, int fd_w, int fd_h, int up, int down)
{
    if (dtype != LVG_F32 && dtype != LVG_F16) return LVG_UNSUPPORTED;
    return pick(fu_w, fu_h, fd_w, fd_h, up, down) == CFG_NONE ? LVG_UNSUPPORTED : LVG_OK;
}

extern "C" int lvg_filtered_lrelu(const void* x, const float* fu, const float* fd, const void* b,
                                  const uint8_t* si, void* y, uint8_t* so, int dtype,
                                  const int64_t x_shape[4], const int64_t x_stride[4],
                                  const int64_t y_shape[4], const int64_t y_stride[4],
                                  int fu_w, int fu_h, int fd_w, int fd_h, int up, int down,
                                  int px0, int py0, int s_h, int s_wbytes, int sx, int sy,
                                  float gain, float slope, float clamp, int flip,
                                  int write_signs, void* stream)
{
    LVG_REQUIRE(x && y && fu && fd && b, "filtered_lrelu: x, y, fu, fd, b must not be NULL");
    LVG_REQUIRE(dtype == LVG_F32 || dtype == LVG_F16, "filtered_lrelu: x must be float16 or float32");
    LVG_REQUIRE(up >= 1 && down >= 1, "filtered_lrelu: up and down must be at least 1");
    for (int i = 0; i < 4; i++) {
        LVG_REQUIRE(x_shape[i] >= 1 && x_shape[i] <= INT32_MAX, "filtered_lrelu: x dimension %d out of range", i);
        LVG_REQUIRE(y_shape[i] >= 1 && y_shape[i] <= INT32_MAX, "filtered_lrelu: output must be at least 1x1");
    }
    LVG_REQUIRE(x_shape[0] == y_shape[0] && x_shape[1] == y_shape[1], "filtered_lrelu: x and y disagree on batch/channels");
    LVG_REQUIRE(y_shape[2] * (y_stride[2] < 0 ? -y_stride[2] : y_stride[2]) < (1ll << 31), "filtered_lrelu: output plane too large");
    LVG_REQUIRE(x_stride[2] >= 0 && x_stride[3] >= 0 &&
                (x_shape[2] + 64) * x_stride[2] + (x_shape[3] + 64) * x_stride[3] < (1ll << 31), "filtered_lrelu: input plane too large");
    LVG_REQUIRE(!(write_signs && si), "filtered_lrelu: cannot read and write signs in one call");
    LVG_REQUIRE(!write_signs || so, "filtered_lrelu: write_signs needs an output sign buffer");
    LVG_REQUIRE(!(write_signs || si) || (s_h >= 1 && s_wbytes >= 1), "filtered_lrelu: bad sign tensor shape");
    const Cfg cfg = pick(fu_w, fu_h, fd_w, fd_h, up, down);
    if (cfg == CFG_NONE) {
        set_error("filtered_lrelu: no fused kernel for up=%d fu=%dx%d down=%d fd=%dx%d", up, fu_w, fu_h, down, fd_w, fd_h);
        return LVG_UNSUPPORTED;
    }

    FlParams p;
    p.x = x; p.fu = fu; p.fd = fd; p.b = b; p.si = si; p.y = y; p.so = so;
    for (int i = 0; i < 4; i++) { p.xs[i] = x_stride[i]; p.ys[i] = y_stride[i]; }
    p.n = (int)x_shape[0]; p.c = (int)x_shape[1]; p.ih = (int)x_shape[2]; p.iw = (int)x_shape[3];
    p.oh = (int)y_shape[2]; p.ow = (int)y_shape[3];
    p.px0 = px0; p.py0 = py0;
    p.s_h = s_h; p.s_wb = s_wbytes; p.sx = sx; p.sy = sy;
    p.sw_active = p.ow * down - (down - 1) + (fd_w - 1);
    p.tiles_x = p.tiles_y = 1;
    p.gain = gain; p.slope = slope; p.clamp = clamp; p.flip = flip ? 1 : 0;
    if (write_signs) {
        // the sign tensor must span the consumed up-sampled extent (filtered_lrelu.cpp:87-94)
        const int need_h = p.oh * down - (down - 1) + ((fd_h ? fd_h : fd_w) - 1);
        LVG_REQUIRE(s_h == need_h && s_wbytes * 4 >= p.sw_active, "filtered_lrelu: sign tensor has the wrong shape");
        LVG_REQUIRE(sx == 0 && sy == 0, "filtered_lrelu: sign offsets only apply when reading signs");
    }
    const int mode = write_signs ? SIGN_WRITE : (si ? SIGN_READ : SIGN_NONE);
    cudaStream_t s = (cudaStream_t)stream;
    return dtype == LVG_F32 ? dispatch<float>(cfg, p, mode, s) : dispatch<__half>(cfg, p, mode, s);
}
