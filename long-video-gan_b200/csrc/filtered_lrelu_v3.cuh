// Fused filtered leaky ReLU, third formulation: every shared-memory access is a 128-bit (or 64-bit)
// access and FMAs come in pairs whose two lanes sit in one aligned register pair as loaded.
//
// Why: a formulation with scalar LDS/STS and per-sample sign codes through a byte tile spends most of its instructions on
// addressing and shared-memory traffic, not on FMAs; here the per-tile instruction count is several times lower and the
// kernel is bounded by shared-memory bandwidth / the FMA pipe instead.
//
// Semantics (torch_utils/ops/filtered_lrelu.cu:139-1099, filtered_lrelu.py:121-153 of the reference):
//   t[U] = up^2 * sum_s gu[s] * z[U + s - pad0],  z = zero-stuffed (x + b), zero outside the image
//   v    = t * gain;  write / plain: v < 0 -> v *= slope (code 1); |v| > clamp -> +-clamp (code 2)
//          read: code = signs[U + sx, V + sy]; bit0 -> v *= slope; bit1 -> v = 0; outside the tensor: unchanged
//   y[o] = sum_t gd[t] * v[o*down + t]
// per axis, separable filters only.
//
// Formulation. The tile's up-sampled axis starts exactly at the first consumed sample U0 = ox0*down (no phase
// alignment slack): up-sampled position c = UP*q + ph (q = "group", ph = phase) is
//     t[c] = sum_{kk <= K} G[ph][kk] * in[q + kk],      K = FU/UP, in[j] = x[M0 + j], M0 = ceil((U0 - pad0)/UP)
// where G[ph] holds the K taps of that phase shifted by e(ph) in {0, 1} and one zero: a (K+1)-tap window that is
// the same for every phase, so register indices are static whatever the padding parity is. G is built per CTA.
//
// Five stages through two shared-memory buffers:
//   1  global -> A_in   [row pair][col][2]                 rows 2p, 2p+1 interleaved (one STS.64 per column)
//   2  up-x:  A_in -> B_ux  (two row-parity planes, row-major)   thread = row pair x 4 groups, FMAs pair the rows
//   3  up-y + gain/lrelu/clamp/signs: B_ux -> A_act          thread = 4 columns x 4 groups, FMAs pair columns;
//        A_act is [row pair m][2 planes][col quad][4]: plane h of quad cg holds columns 4cg+2h, +1 of both rows, so the
//        writer's lanes store consecutive 16-byte pieces and the reader gets (row a, row b) pairs by LDS.128.
//        A row pair is (UP*(2qq) + ph, UP*(2qq+1) + ph) -- the two rows one thread produces with ONE set of taps.
//        One sign byte = the thread's 4 columns: stored straight to global (write) / one table lookup (read).
//   4  down-x: A_act -> B_dx (two planes by pair slot)       thread = row pair x RDX outputs, FMAs pair the rows
//   5  down-y: B_dx -> global                                 thread = 2 columns x RDY outputs, FMAs pair columns
// Pitches are chosen so that each quarter warp of every 128-bit access covers all 32 banks once.
//
// The stage functions take the thread index as an argument and contain no warp-level primitives, so the same
// source compiles as host code (FLV3_HOST_EMU) where the stages run thread by thread -- tools/fl_emul.cu checks
// the index arithmetic against the operator's definition on the CPU.

#pragma once
#include <cuda_fp16.h>
#include <stdint.h>
#include <math.h>
#include <string.h>
#ifdef FLV3_HOST_EMU
#include <assert.h>
#include <vector_types.h>
#include <vector_functions.h>
#define FL_HD inline
#else
#define FL_HD __device__ __forceinline__
#endif

namespace lvg {
namespace flv3 {

enum { SIGN_NONE = 0, SIGN_WRITE = 1, SIGN_READ = 2 };
constexpr int kThreads = 256;

struct FlParams {
    const void* x;
    const float* fu;
    const float* fd;
    const void* b;
    const uint8_t* si;
    void* y;
    uint8_t* so;
    int64_t xs[4], ys[4];
    int n, c, ih, iw, oh, ow;
    int px0, py0;
    int s_h, s_wb, sx, sy;
    int sw_active;          // write mode: samples at U >= sw_active get code 0
    int tiles_x, tiles_y;
    float gain, slope, clamp;
    int flip;
    // launch constants prepared by the host (fill_launch_constants)
    float tap_scale;                 // sqrt(up^2 * gain): folded into each of the two up-sampling passes
    int cpx, cpy;                    // first input sample of a tile: U0/UP + cpx (U0 is a multiple of UP)
    unsigned mg_tiles, mg_tx, mg_c;  // ceil(2^32 / d) for the block-index decomposition
    signed char gx_idx[32], gy_idx[32];   // padded phase windows: index into the up filter, -1 = zero tap
};

constexpr int cdiv(int a, int b) { return (a + b - 1) / b; }
constexpr int rup(int a, int b) { return cdiv(a, b) * b; }
constexpr int cmax(int a, int b) { return a > b ? a : b; }
constexpr int pitch_mod(int w, int m, int r) { int p = w; while (p % m != r) p++; return p; }

FL_HD int imin(int a, int b) { return a < b ? a : b; }
FL_HD int imax(int a, int b) { return a > b ? a : b; }
FL_HD int fdiv_floor(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
FL_HD int fdiv_ceil(int a, int b) { return fdiv_floor(a + b - 1, b); }

// ---- memory and arithmetic primitives (device: vector LDS/STS and paired FMAs; host: plain C with alignment asserts)
FL_HD float4 lds4(const float* p)
{
#ifdef FLV3_HOST_EMU
    assert(((uintptr_t)p & 15) == 0);
#endif
    return *reinterpret_cast<const float4*>(p);
}
FL_HD float2 lds2(const float* p)
{
#ifdef FLV3_HOST_EMU
    assert(((uintptr_t)p & 7) == 0);
#endif
    return *reinterpret_cast<const float2*>(p);
}
FL_HD void sts4(float* p, float a, float b, float c, float d)
{
#ifdef FLV3_HOST_EMU
    assert(((uintptr_t)p & 15) == 0);
#endif
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
FL_HD void sts2(float* p, float a, float b)
{
#ifdef FLV3_HOST_EMU
    assert(((uintptr_t)p & 7) == 0);
#endif
    *reinterpret_cast<float2*>(p) = make_float2(a, b);
}
FL_HD float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
template <class T> FL_HD float ld_as_float(const T* p);
template <> FL_HD float ld_as_float<float>(const float* p) { return *p; }
template <> FL_HD float ld_as_float<__half>(const __half* p) { return __half2float(*p); }
// x + bias in fp32
FL_HD float ld_plus(const float* p, float bias) { return *p + bias; }
FL_HD float ld_plus(const __half* p, float bias)
{
#ifdef FLV3_HOST_EMU
    return __half2float(*p) + bias;
#else
    return __half2float(*p) + bias;
#endif
}
// x[i] + bias with the element address formed by ONE wide multiply-add (the compiler otherwise spends four
// instructions per 64-bit element address)
FL_HD float ld_plus_at(const float* p, int i, float bias)
{
#ifdef FLV3_HOST_EMU
    return p[i] + bias;
#else
    float r;
    asm("{ .reg .b64 a; .reg .f32 v; mad.wide.s32 a, %1, 4, %2; ld.global.nc.f32 v, [a]; add.rn.f32 %0, v, %3; }"
        : "=f"(r) : "r"(i), "l"(p), "f"(bias));
    return r;
#endif
}
FL_HD float ld_plus_at(const __half* p, int i, float bias)
{
#ifdef FLV3_HOST_EMU
    return __half2float(p[i]) + bias;
#else
    float r;
    asm("{ .reg .b64 a; .reg .b16 h; .reg .f32 v; mad.wide.s32 a, %1, 2, %2; ld.global.nc.b16 h, [a]; cvt.f32.f16 v, h; add.rn.f32 %0, v, %3; }"
        : "=f"(r) : "r"(i), "l"(p), "f"(bias));
    return r;
#endif
}
// if (ok) *q = v as a predicated store (no branch around it)
FL_HD void st_byte_if(uint8_t* q, bool ok, unsigned v)
{
#ifdef FLV3_HOST_EMU
    if (ok) *q = (uint8_t)v;
#else
    asm volatile("{ .reg .pred p; setp.ne.s32 p, %1, 0; @p st.global.u8 [%0], %2; }" :: "l"(q), "r"((int)ok), "r"(v) : "memory");
#endif
}
FL_HD float2 mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
// bits 2k of the result = sign bits of v[k] (k < 4); higher bits are garbage the caller masks away.
// Two byte permutes gather the four top bytes, one multiply moves bit 8k+7 to bit 32+2k.
FL_HD unsigned sign_bits4(float v0, float v1, float v2, float v3)
{
#ifdef FLV3_HOST_EMU
    unsigned u[4]; float f[4] = {v0, v1, v2, v3}; memcpy(u, f, 16);
    return (u[0] >> 31) | ((u[1] >> 31) << 2) | ((u[2] >> 31) << 4) | ((u[3] >> 31) << 6);
#else
    const unsigned t0 = __byte_perm(__float_as_uint(v0), __float_as_uint(v1), 0x0073);
    const unsigned t1 = __byte_perm(__float_as_uint(v2), __float_as_uint(v3), 0x0073);
    const unsigned w = __byte_perm(t0, t1, 0x5410) & 0x80808080u;
    return __umulhi(w, (1u << 25) + (1u << 19) + (1u << 13) + (1u << 7));
#endif
}
FL_HD unsigned fbits(float v)
{
#ifdef FLV3_HOST_EMU
    unsigned u; memcpy(&u, &v, 4); return u;
#else
    return __float_as_uint(v);
#endif
}
// n / d with magic = ceil(2^32 / d); exact for n * d < 2^32 (the host checks the grid against that)
FL_HD unsigned udiv(unsigned n, unsigned d, unsigned magic)
{
#ifdef FLV3_HOST_EMU
    (void)magic; return n / d;
#else
    return d > 1 ? __umulhi(n, magic) : n;
#endif
}
template <class T> FL_HD void st_from_float(T* p, float v);
template <> FL_HD void st_from_float<float>(float* p, float v) { *p = v; }
template <> FL_HD void st_from_float<__half>(__half* p, float v) { *p = __float2half_rn(v); }

// n / d for the item indices of a stage (n < 2^15, d < 2^10): (n + 0.5) * (1/d) truncated. (n + 0.5)/d is at least 0.5/d
// away from an integer, far more than the rounding error of the reciprocal, so the quotient is exact -- three
// instructions per use and one reciprocal per stage instead of the 32-bit division sequence.
struct FastDiv {
    float inv;
    int d;
    FL_HD explicit FastDiv(int d_) : inv(1.0f / (float)d_), d(d_) {}
    FL_HD int div(int n) const
    {
#ifdef FLV3_HOST_EMU
        const int q = (int)(((float)n + 0.5f) * inv);
        assert(q == n / d);
        return q;
#else
        return __float2int_rz(((float)n + 0.5f) * inv);
#endif
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// RX, RY: groups per thread in the up passes; RDX, RDY: outputs per thread in the down passes. They set the number of
// work items of each stage: chosen per configuration so that a stage is (close to) ONE round over the CTA's 256 threads --
// a second, nearly empty round leaves most warps waiting at the barrier.
template <int UP_, int FU_, int DOWN_, int FD_, int TOW_, int TOH_, int RX_, int RY_, int RDX_, int RDY_>
struct Geom {
    static constexpr int UP = UP_, FU = FU_, DOWN = DOWN_, FD = FD_, TOW = TOW_, TOH = TOH_, RDX = RDX_, RDY = RDY_;
    static constexpr int K = FU / UP, KT = K + 1;          // taps per phase, padded window
    static constexpr int RX = RX_, RY = RY_;
    static constexpr int TUW = (TOW - 1) * DOWN + FD, TUH = (TOH - 1) * DOWN + FD;     // consumed up-sampled extent
    static constexpr int NQXR = rup(cdiv(TUW, UP), RX), NQYR = rup(cdiv(TUH, UP), RY);
    static constexpr int UW = NQXR * UP, UH = NQYR * UP;   // computed up-sampled extent
    static constexpr int VX = rup(RX + K, 4);              // input columns one thread of the x up pass loads
    static constexpr int TIW = NQXR + K, TIH = NQYR + K;   // input tile
    static constexpr int NRP_IN = TIH / 2;
    static constexpr int P_IN = pitch_mod(NQXR - RX + VX, 4, 2);
    static constexpr int S_IN = 2 * P_IN;                  // words per row pair, S_IN/4 odd
    static constexpr int A_IN = NRP_IN * S_IN;
    static constexpr int P_UX = pitch_mod(UW, 8, 4);
    static constexpr int PL_UX = NRP_IN * P_UX;
    static constexpr int B_UX = 2 * PL_UX;
    static constexpr int NINX = (RDX - 1) * DOWN + FD, NINXP = rup(NINX, 4);
    static constexpr int NTD = cdiv(TOW, RDX);
    static constexpr int DX_EXT = DOWN * RDX * (NTD - 1) + NINXP;
    static constexpr int NCG = cdiv(cmax(UW, DX_EXT), 4);
    static constexpr int HS = NCG * 4;                     // plane stride inside a row pair
    static constexpr int S_A = 2 * HS + 4;                 // words per row pair, S_A/4 odd
    static constexpr int NRP_A = UH / 2;
    static constexpr int A_ACT = NRP_A * S_A;
    static constexpr int P_DX = RDX == 4 ? pitch_mod(rup(TOW, 4), 8, 4) : pitch_mod(rup(TOW, 2), 4, 2);
    static constexpr int NRP_D = rup(TUH, 2 * UP) / 2;
    static constexpr int PL_DX = rup(NRP_D * P_DX, 4);
    static constexpr int B_DX = 2 * PL_DX;
    static constexpr int NINY = (RDY - 1) * DOWN + FD;
    static constexpr int A_SIZE = cmax(A_IN, A_ACT), B_SIZE = cmax(B_UX, B_DX);
    static constexpr int TAPS = 2 * (2 * UP * KT) + 2 * FD + 32;      // gx pairs, gy pairs, fd pairs, sign multiplier table
    static constexpr int SIGN_PITCH = rup(UW / 4 + 2 + 3, 4);        // staged bytes per row: a thread's two bytes + word-alignment slack
    static constexpr int SIGN_BYTES = rup(UH * SIGN_PITCH, 16);
    static constexpr bool STREAM_TAPS = FD > 12;           // 24-tap down filters: taps read per use instead of held in registers
    static_assert(FU % UP == 0 && K % 2 == 0, "filter length must be an even multiple of the up-sampling factor");
    static_assert((DOWN * RDY) % (2 * UP) == 0, "row groups of the last pass must start on a row-pair block");
    static_assert((DOWN * RDX) % 4 == 0 && (TOW * DOWN) % 4 == 0, "column groups must start on a column quad");
    static_assert(RDX == 2 || RDX == 4, "RDX");
    static_assert(UW % 4 == 0 && UH % (2 * UP) == 0 && TIH % 2 == 0 && RY % 2 == 0 && (RX * UP) % 4 == 0, "extents");
    static constexpr size_t smem_bytes(int mode)
    {
        return (size_t)(A_SIZE + B_SIZE + TAPS) * sizeof(float) + (mode == SIGN_READ ? SIGN_BYTES : 0);
    }
    // resident CTAs per SM the kernel is compiled for (227 KB of shared memory per SM, 1 KB reserved per CTA). Four CTAs
    // mean 64 registers per thread: the up-4 configuration fits without spilling, up-2 / down-2 spills 60-140 bytes.
    static constexpr int ctas(int mode)
    {
        const int bytes = (A_SIZE + B_SIZE + TAPS) * 4 + (mode == SIGN_READ ? SIGN_BYTES : 0) + 1024;
        return bytes * 4 <= 232448 ? 4 : bytes * 3 <= 232448 ? 3 : 2;
    }
};

struct Tile {
    int nn, cc, tx, ty;
    unsigned plane;
    int ox0, oy0, U0, V0;
    int m0x, m0y;                 // first input sample of the tile
    int tow_e, toh_e, tuw_e, tuh_e;
    int ntg_e, ntgy_e;            // thread-level group counts of the up passes
    int tiw_e, tih_e, nrp_e, ncg_e, uh_e;
};

template <class G>
FL_HD Tile make_tile(const FlParams& p, unsigned bid)
{
    Tile t;
    const unsigned tiles = (unsigned)(p.tiles_x * p.tiles_y);
    t.plane = udiv(bid, tiles, p.mg_tiles);
    const unsigned tile = bid - t.plane * tiles;
    t.ty = (int)udiv(tile, (unsigned)p.tiles_x, p.mg_tx);
    t.tx = (int)tile - t.ty * p.tiles_x;
    t.nn = (int)udiv(t.plane, (unsigned)p.c, p.mg_c);
    t.cc = (int)(t.plane - (unsigned)t.nn * (unsigned)p.c);
    t.ox0 = t.tx * G::TOW; t.oy0 = t.ty * G::TOH;
    t.U0 = t.ox0 * G::DOWN; t.V0 = t.oy0 * G::DOWN;
    t.m0x = t.U0 / G::UP + p.cpx; t.m0y = t.V0 / G::UP + p.cpy;        // = ceil((U0 - pad0) / UP)
    t.tow_e = imin(G::TOW, p.ow - t.ox0); t.toh_e = imin(G::TOH, p.oh - t.oy0);
    t.tuw_e = (t.tow_e - 1) * G::DOWN + G::FD; t.tuh_e = (t.toh_e - 1) * G::DOWN + G::FD;
    t.ntg_e = cdiv(cdiv(t.tuw_e, G::UP), G::RX); t.ntgy_e = cdiv(cdiv(t.tuh_e, G::UP), G::RY);
    t.tiw_e = t.ntg_e * G::RX + G::K; t.tih_e = t.ntgy_e * G::RY + G::K;
    t.nrp_e = t.tih_e / 2;
    t.ncg_e = cdiv(t.tuw_e, 4);                     // column quads the later stages consume (<= the columns stage 2 computes)
    t.uh_e = t.ntgy_e * G::RY * G::UP;
    return t;
}

// Host side: tile counts, block-index magics and the padded phase windows (see the header comment). U0 = tx*TOW*DOWN is
// a multiple of UP, so the windows depend on the padding only and are the same for every tile.
template <class G>
inline void fill_launch_constants(FlParams& p)
{
    p.tiles_x = cdiv(p.ow, G::TOW);
    p.tiles_y = cdiv(p.oh, G::TOH);
    p.tap_scale = sqrtf((float)(G::UP * G::UP) * p.gain);
    auto magic = [](unsigned d) { return d > 1 ? 0xFFFFFFFFu / d + 1u : 0u; };
    p.mg_tiles = magic((unsigned)(p.tiles_x * p.tiles_y));
    p.mg_tx = magic((unsigned)p.tiles_x);
    p.mg_c = magic((unsigned)p.c);
    auto ceil_div = [](int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) == (b < 0))) ? q + 1 : q; };
    for (int axis = 0; axis < 2; axis++) {
        const int d = -(axis ? p.py0 : p.px0);
        const int m0 = ceil_div(d, G::UP);
        (axis ? p.cpy : p.cpx) = m0;
        for (int ph = 0; ph < G::UP; ph++) {
            const int cph = ceil_div(d + ph, G::UP), e = cph - m0, s0 = G::UP * cph - (d + ph);
            for (int kk = 0; kk < G::KT; kk++) {
                const int k = kk - e;
                (axis ? p.gy_idx : p.gx_idx)[ph * G::KT + kk] = (signed char)((k >= 0 && k < G::K) ? s0 + k * G::UP : -1);
            }
        }
    }
}

struct Smem {
    float *A, *B, *gx, *gy, *fd2, *lut;
    uint8_t* sign;
};

template <class G>
FL_HD Smem carve(float* smem)
{
    Smem s;
    s.A = smem;
    s.B = s.A + G::A_SIZE;
    s.gx = s.B + G::B_SIZE;
    s.gy = s.gx + 2 * G::UP * G::KT;
    s.fd2 = s.gy + 2 * G::UP * G::KT;
    s.lut = s.fd2 + 2 * G::FD;
    s.sign = reinterpret_cast<uint8_t*>(s.lut + 32);
    return s;
}

// ---- stage 0: per-tile tap tables, sign multiplier table, and (read mode) this tile's slab of the sign tensor
template <class G, int MODE>
FL_HD void stage0(const FlParams& p, const Tile& t, const Smem& s, int tid)
{
    // padded phase windows of the up filter from the host's index tables (taps arrive as device pointers)
    for (int idx = tid; idx < 2 * G::UP * G::KT; idx += kThreads) {
        const int axis = idx >= G::UP * G::KT, r = idx - axis * (G::UP * G::KT);
        const int i = axis ? p.gy_idx[r] : p.gx_idx[r];
        const float v = i < 0 ? 0.f : (p.flip ? p.fu[i] : p.fu[G::FU - 1 - i]) * p.tap_scale;
        float* dst = (axis ? s.gy : s.gx) + 2 * r;
        dst[0] = v; dst[1] = v;
    }
    for (int i = tid; i < G::FD; i += kThreads) {
        const float v = p.flip ? p.fd[i] : p.fd[G::FD - 1 - i];
        s.fd2[2 * i] = v; s.fd2[2 * i + 1] = v;
    }
    if (MODE == SIGN_READ) {
        for (int i = tid; i < 32; i += kThreads) {
            const int c = (i & 1) ? ((i >> 1) >> 2) : ((i >> 1) & 3);          // entry n = i/2 holds the multipliers of codes n&3, n>>2
            s.lut[i] = (c & 2) ? 0.f : ((c & 1) ? p.slope : 1.f);
        }
        // the tile's slab of the sign tensor, staged with aligned 32-bit loads (rows are multiples of 4 bytes, host-checked):
        // staged row r holds global bytes [gb_al, gb_al + SIGN_PITCH) of row V0 + sy + r, gb_al = first needed byte rounded down
        const uint8_t* sgn = p.si + t.plane * (int64_t)p.s_h * p.s_wb;
        const int gy0 = t.V0 + p.sy, gb_al = ((t.U0 + p.sx) >> 2) & ~3;         // arithmetic shift / mask = floor
        constexpr int W4 = G::SIGN_PITCH / 4;
        uint32_t* dst = reinterpret_cast<uint32_t*>(s.sign);
        for (int i = tid; i < t.uh_e * W4; i += kThreads) {
            const int row = i / W4, w = i - row * W4;
            const int gy = gy0 + row, gb = gb_al + 4 * w;
            uint32_t v = 0;
            if ((unsigned)gy < (unsigned)p.s_h && (unsigned)gb < (unsigned)p.s_wb)
                v = *reinterpret_cast<const uint32_t*>(sgn + (int64_t)gy * p.s_wb + gb);
            dst[i] = v;
        }
    }
}

// ---- stage 1: input tile (+ bias inside the image, zero outside) -> A_in[row pair][col][2]
// One warp per row pair, lanes along the row; fully unrolled, all global loads of a thread are issued before the first
// shared-memory store. Rows are uniform per warp (a row outside the image costs no loads), columns are a per-lane
// predicate computed once; an element costs an address add, the load, one mixed-precision add (bias) and a select.
template <class T, class G>
FL_HD void stage1(const FlParams& p, const Tile& t, const Smem& s, int tid)
{
    const T* xp = (const T*)p.x + (int64_t)t.nn * p.xs[0] + (int64_t)t.cc * p.xs[1];
    const float bias = ld_plus((const T*)p.b + t.cc, 0.f);
    constexpr int kWarps = kThreads / 32;
    constexpr int kRowIters = cdiv(G::NRP_IN, kWarps), kColIters = cdiv(G::TIW, 32);
    const int warp = tid / 32, lane = tid % 32;
    const int xs2 = (int)p.xs[2], xs3 = (int)p.xs[3];      // offsets inside one (n, c) plane fit 32 bits (host check)
    // Loads are unconditional from coordinates clamped into the image (no branches, no predicated loads); samples
    // outside the image are then replaced by zero (two selects: the column predicate per lane, the row predicate per warp).
    bool colok[kColIters];
    const T* colp[kColIters];                              // column pointers: an element address is one wide multiply-add
#pragma unroll
    for (int cj = 0; cj < kColIters; cj++) {
        const int gx = t.m0x + lane + 32 * cj;
        colok[cj] = (unsigned)gx < (unsigned)p.iw;
        colp[cj] = xp + imin(imax(gx, 0), p.iw - 1) * xs3;
    }
    float v[kRowIters][kColIters][2];
#pragma unroll
    for (int ri = 0; ri < kRowIters; ri++) {
        const int rp = warp + kWarps * ri;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int gy = t.m0y + 2 * rp + h;
            const bool rowok = (unsigned)gy < (unsigned)p.ih;
            const int rowoff = imin(imax(gy, 0), p.ih - 1) * xs2;
#pragma unroll
            for (int cj = 0; cj < kColIters; cj++) {
                const float x = ld_plus_at(colp[cj], rowoff, bias);
                v[ri][cj][h] = (rowok && colok[cj]) ? x : 0.f;
            }
        }
    }
#pragma unroll
    for (int ri = 0; ri < kRowIters; ri++) {
        const int rp = warp + kWarps * ri;
        if (rp < G::NRP_IN) {
#pragma unroll
            for (int cj = 0; cj < kColIters; cj++) {
                const int ix = lane + 32 * cj;
                if (ix < G::TIW) sts2(s.A + rp * G::S_IN + 2 * ix, v[ri][cj][0], v[ri][cj][1]);
            }
        }
    }
}

// ---- stage 2: up-sample along x.  A_in -> B_ux[row parity][row/2][col]
template <class G>
FL_HD void stage2(const Tile& t, const Smem& s, int tid)
{
    constexpr int UP = G::UP, KT = G::KT, RX = G::RX;
    const int nitems = t.nrp_e * t.ntg_e;
    const FastDiv by_rp(t.nrp_e);
#pragma unroll 1
    for (int id = tid; id < nitems; id += kThreads) {
        const int tg = by_rp.div(id), rp = id - tg * t.nrp_e;
        const float* src = s.A + rp * G::S_IN + 2 * RX * tg;
        float2 v[G::VX];
#pragma unroll
        for (int j = 0; j < G::VX / 2; j++) {
            const float4 l = lds4(src + 4 * j);
            v[2 * j] = make_float2(l.x, l.y);
            v[2 * j + 1] = make_float2(l.z, l.w);
        }
        float2 acc[RX * UP];
#pragma unroll
        for (int ph = 0; ph < UP; ph++) {
            float2 g[KT];
#pragma unroll
            for (int kk = 0; kk < KT; kk++) g[kk] = lds2(s.gx + 2 * (ph * KT + kk));
#pragma unroll
            for (int q = 0; q < RX; q++) {
                float2 a = make_float2(0.f, 0.f);
#pragma unroll
                for (int kk = 0; kk < KT; kk++) a = fma2(g[kk], v[q + kk], a);
                acc[q * UP + ph] = a;
            }
        }
        float* d0 = s.B + rp * G::P_UX + RX * UP * tg;
        float* d1 = d0 + G::PL_UX;
#pragma unroll
        for (int j = 0; j < RX * UP / 4; j++) {
            sts4(d0 + 4 * j, acc[4 * j].x, acc[4 * j + 1].x, acc[4 * j + 2].x, acc[4 * j + 3].x);
            sts4(d1 + 4 * j, acc[4 * j].y, acc[4 * j + 1].y, acc[4 * j + 2].y, acc[4 * j + 3].y);
        }
    }
}

// ---- stage 3: up-sample along y, activation, signs.  B_ux -> A_act
// Activation cost matters here (7 FMAs per sample only): the leaky ReLU is max/min(v, v*slope), the clamp and the
// "clamped" code are skipped for a thread's 8 samples at once when none of them exceeds the clamp (one max tree, one
// compare), and the "negative" code bits are the sign bits of the raw values (an accumulator that starts at +0 never
// becomes -0 under round-to-nearest, so sign bit <=> v < 0).
template <class G, int MODE>
FL_HD void stage3(const FlParams& p, const Tile& t, const Smem& s, int tid)
{
    constexpr int UP = G::UP, KT = G::KT, RY = G::RY, NV = G::K + G::RY;
    const float slope = p.slope, clamp = p.clamp;
    const float2 slope2 = make_float2(slope, slope);       // slope <= 1 (host-checked): lrelu(v) = max(v, v*slope)
    // write mode: this CTA's byte-aligned slab of the sign tensor
    const bool lastx = (t.tx == p.tiles_x - 1), lasty = (t.ty == p.tiles_y - 1);
    const int b0 = t.U0 >> 2;
    const int nb = (lastx ? p.s_wb : imin(p.s_wb, (t.U0 + G::TOW * G::DOWN) >> 2)) - b0;
    const int nr = (lasty ? p.s_h : imin(p.s_h, t.V0 + G::TOH * G::DOWN)) - t.V0;
    uint8_t* so = MODE == SIGN_WRITE ? p.so + t.plane * (int64_t)p.s_h * p.s_wb + (int64_t)t.V0 * p.s_wb + b0 : nullptr;
    const int s_wb = p.s_wb;
    const int sh2 = ((t.U0 + p.sx) & 3) * 2;                // read mode: bit offset of the first sample inside its byte
    const int sgn_skew = ((t.U0 + p.sx) >> 2) & 3;          //            first needed byte inside the staged (word-aligned) row

    const int nitems = t.ncg_e * t.ntgy_e;
    const FastDiv by_cg(t.ncg_e);
#pragma unroll 1
    for (int id = tid; id < nitems; id += kThreads) {
        const int tgy = by_cg.div(id), cg = id - tgy * t.ncg_e;
        const float* src = s.B + (tgy * (RY / 2)) * G::P_UX + 4 * cg;
        float4 v[NV];
#pragma unroll
        for (int i = 0; i < NV; i++) v[i] = lds4(src + (i & 1) * G::PL_UX + (i >> 1) * G::P_UX);
        uint8_t* so_item = nullptr;
        int rows_left = 0;                                   // sign rows of this item inside the slab
        if (MODE == SIGN_WRITE) {
            so_item = so + (tgy * RY * UP) * s_wb + cg;
            rows_left = cg < nb ? nr - tgy * RY * UP : 0;
        }
        float* dst_item = s.A + (tgy * (RY / 2) * UP) * G::S_A + 4 * cg;
        const uint8_t* sr_item = MODE == SIGN_READ ? s.sign + (tgy * RY * UP) * G::SIGN_PITCH + cg + sgn_skew : nullptr;
#pragma unroll
        for (int ph = 0; ph < UP; ph++) {
            float2 g[KT];
#pragma unroll
            for (int kk = 0; kk < KT; kk++) g[kk] = lds2(s.gy + 2 * (ph * KT + kk));
#pragma unroll
            for (int jp = 0; jp < RY / 2; jp++) {
                float2 a[2][2];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    a[h][0] = make_float2(0.f, 0.f); a[h][1] = make_float2(0.f, 0.f);
#pragma unroll
                    for (int kk = 0; kk < KT; kk++) {
                        const float4 w = v[2 * jp + h + kk];
                        a[h][0] = fma2(g[kk], make_float2(w.x, w.y), a[h][0]);
                        a[h][1] = fma2(g[kk], make_float2(w.z, w.w), a[h][1]);
                    }
                }
                float o[2][4];
                if (MODE == SIGN_READ) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const uint8_t* sr = sr_item + ((2 * jp + h) * UP + ph) * G::SIGN_PITCH;
                        const unsigned c8 = (((unsigned)sr[0] | ((unsigned)sr[1] << 8)) >> sh2) & 0xFFu;
                        const float2 m0 = lds2(s.lut + 2 * (c8 & 15u)), m1 = lds2(s.lut + 2 * (c8 >> 4));
                        o[h][0] = a[h][0].x * m0.x; o[h][1] = a[h][0].y * m0.y; o[h][2] = a[h][1].x * m1.x; o[h][3] = a[h][1].y * m1.y;
                    }
                } else {
                    // leaky ReLU on all 8 samples, then ONE test whether any of them needs the clamp
                    float mx = 0.f;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
#pragma unroll
                        for (int c2 = 0; c2 < 2; c2++) {
                            const float2 r = a[h][c2], rs = mul2(r, slope2);
                            const float l0 = fmaxf(r.x, rs.x), l1 = fmaxf(r.y, rs.y);
                            o[h][2 * c2] = l0; o[h][2 * c2 + 1] = l1;
                            mx = fmaxf(mx, fmaxf(fabsf(l0), fabsf(l1)));
                        }
                    }
                    unsigned byte[2];
                    if (MODE == SIGN_WRITE) {
#pragma unroll
                        for (int h = 0; h < 2; h++)
                            byte[h] = sign_bits4(a[h][0].x, a[h][0].y, a[h][1].x, a[h][1].y);
                    }
                    if (mx > clamp) {                        // rare: some sample saturates
#pragma unroll
                        for (int h = 0; h < 2; h++) {
#pragma unroll
                            for (int k = 0; k < 4; k++) {
                                const float l = o[h][k];
                                if (fabsf(l) > clamp) {
                                    o[h][k] = l < 0.f ? -clamp : clamp;
                                    if (MODE == SIGN_WRITE) byte[h] = (byte[h] & ~(3u << (2 * k))) | (2u << (2 * k));
                                }
                            }
                        }
                    }
                    if (MODE == SIGN_WRITE) {
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int rl = (2 * jp + h) * UP + ph;
                            st_byte_if(so_item + rl * s_wb, rl < rows_left, byte[h]);
                        }
                    }
                }
                float* dst = dst_item + (jp * UP + ph) * G::S_A;          // row pair m = (tgy*RY/2 + jp)*UP + ph
                sts4(dst, o[0][0], o[1][0], o[0][1], o[1][1]);
                sts4(dst + G::HS, o[0][2], o[1][2], o[0][3], o[1][3]);
            }
        }
    }
    // write mode, last tile of a row: the sign tensor's width is padded to 16 samples; bytes beyond the computed columns are zero
    if (MODE == SIGN_WRITE && nb > t.ncg_e) {
        const int extra = nb - t.ncg_e;
        for (int i = tid; i < extra * nr; i += kThreads) {
            const int row = i / extra, bb = i - row * extra;
            so[(int64_t)row * s_wb + t.ncg_e + bb] = 0;
        }
    }
}

// write mode, after the barrier that follows stage 3: samples at U >= sw_active carry code 0. Only the byte that straddles
// sw_active in the last tile of a row can hold such samples; it is masked here instead of in the inner loop.
template <class G>
FL_HD void stage3_fixup(const FlParams& p, const Tile& t, int tid)
{
    const int na = p.sw_active - t.U0;                      // active samples from the tile's first column
    if (t.tx != p.tiles_x - 1 || (na & 3) == 0 || na <= 0 || (na >> 2) >= t.ncg_e) return;
    const bool lasty = (t.ty == p.tiles_y - 1);
    const int nr = (lasty ? p.s_h : imin(p.s_h, t.V0 + G::TOH * G::DOWN)) - t.V0;
    uint8_t* so = p.so + t.plane * (int64_t)p.s_h * p.s_wb + (int64_t)t.V0 * p.s_wb + (t.U0 >> 2) + (na >> 2);
    const unsigned mask = (1u << (2 * (na & 3))) - 1u;
    for (int row = tid; row < nr; row += kThreads) so[(int64_t)row * p.s_wb] &= (uint8_t)mask;
}

// ---- stage 4: down-sample along x.  A_act -> B_dx[pair slot][pair][col]
template <class G>
FL_HD void stage4(const Tile& t, const Smem& s, int tid)
{
    constexpr int DOWN = G::DOWN, FD = G::FD, RDX = G::RDX;
    float2 g[G::STREAM_TAPS ? 1 : FD];
    if (!G::STREAM_TAPS) {
#pragma unroll
        for (int i = 0; i < FD; i++) g[i] = lds2(s.fd2 + 2 * i);
    }
    const int nm_e = cdiv(t.tuh_e, 2 * G::UP) * G::UP;
    const int ntd_e = cdiv(t.tow_e, RDX);
    const FastDiv by_m(nm_e);
#pragma unroll 1
    for (int id = tid; id < nm_e * ntd_e; id += kThreads) {
        const int tgd = by_m.div(id), m = id - tgd * nm_e;
        const float* src = s.A + m * G::S_A + DOWN * RDX * tgd;
        float2 v[G::NINXP];
#pragma unroll
        for (int j = 0; j < G::NINXP / 2; j++) {
            const float4 l = lds4(src + (j & 1) * G::HS + 4 * (j >> 1));
            v[2 * j] = make_float2(l.x, l.y);
            v[2 * j + 1] = make_float2(l.z, l.w);
        }
        float2 acc[RDX];
#pragma unroll
        for (int o = 0; o < RDX; o++) acc[o] = make_float2(0.f, 0.f);
        if (G::STREAM_TAPS) {
#pragma unroll
            for (int tt = 0; tt < FD; tt++) {
                const float2 gt = lds2(s.fd2 + 2 * tt);
#pragma unroll
                for (int o = 0; o < RDX; o++) acc[o] = fma2(gt, v[o * DOWN + tt], acc[o]);
            }
        } else {
#pragma unroll
            for (int o = 0; o < RDX; o++) {
#pragma unroll
                for (int tt = 0; tt < FD; tt++) acc[o] = fma2(g[tt], v[o * DOWN + tt], acc[o]);
            }
        }
        float* d0 = s.B + m * G::P_DX + RDX * tgd;
        float* d1 = d0 + G::PL_DX;
        if (RDX == 4) {
            sts4(d0, acc[0].x, acc[1].x, acc[2].x, acc[3].x);
            sts4(d1, acc[0].y, acc[1].y, acc[2].y, acc[3].y);
        } else {
            sts2(d0, acc[0].x, acc[1].x);
            sts2(d1, acc[0].y, acc[1].y);
        }
    }
}

// ---- stage 5: down-sample along y and store
template <class T, class G>
FL_HD void stage5(const FlParams& p, const Tile& t, const Smem& s, int tid)
{
    constexpr int DOWN = G::DOWN, FD = G::FD, RDY = G::RDY, UP = G::UP;
    float2 g[G::STREAM_TAPS ? 1 : FD];
    if (!G::STREAM_TAPS) {
#pragma unroll
        for (int i = 0; i < FD; i++) g[i] = lds2(s.fd2 + 2 * i);
    }
    T* yp = (T*)p.y + (int64_t)t.nn * p.ys[0] + (int64_t)t.cc * p.ys[1] + (int64_t)t.oy0 * p.ys[2] + (int64_t)t.ox0 * p.ys[3];
    const int ys2 = (int)p.ys[2], ys3 = (int)p.ys[3];      // a plane spans < 2^31 elements (host check)
    const int ncp_e = cdiv(t.tow_e, 2), ntg5_e = cdiv(t.toh_e, RDY);
    const FastDiv by_cp(ncp_e);
#pragma unroll 1
    for (int id = tid; id < ncp_e * ntg5_e; id += kThreads) {
        const int tg5 = by_cp.div(id), cp = id - tg5 * ncp_e;
        const int mb = (DOWN * RDY * tg5) / (2 * UP) * UP;
        const float* src = s.B + mb * G::P_DX + 2 * cp;
        float2 v[G::NINY];
#pragma unroll
        for (int i = 0; i < G::NINY; i++)
            v[i] = lds2(src + ((i / UP) & 1) * G::PL_DX + ((i / (2 * UP)) * UP + i % UP) * G::P_DX);
        float2 acc[RDY];
#pragma unroll
        for (int o = 0; o < RDY; o++) acc[o] = make_float2(0.f, 0.f);
        if (G::STREAM_TAPS) {
#pragma unroll
            for (int tt = 0; tt < FD; tt++) {
                const float2 gt = lds2(s.fd2 + 2 * tt);
#pragma unroll
                for (int o = 0; o < RDY; o++) acc[o] = fma2(gt, v[o * DOWN + tt], acc[o]);
            }
        } else {
#pragma unroll
            for (int o = 0; o < RDY; o++) {
#pragma unroll
                for (int tt = 0; tt < FD; tt++) acc[o] = fma2(g[tt], v[o * DOWN + tt], acc[o]);
            }
        }
        const bool two = 2 * cp + 1 < t.tow_e;
        T* q = yp + 2 * cp * ys3;
#pragma unroll
        for (int o = 0; o < RDY; o++) {
            const int oy = RDY * tg5 + o;
            if (oy < t.toh_e) {
                st_from_float(q + oy * ys2, acc[o].x);
                if (two) st_from_float(q + oy * ys2 + ys3, acc[o].y);
            }
        }
    }
}

}  // namespace flv3
}  // namespace lvg
