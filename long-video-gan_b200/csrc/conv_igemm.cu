// Grouped 1-D / 2-D / 3-D convolution (cross-correlation) as a TMA-fed implicit GEMM on Hopper tensor cores (wgmma).
//
// One engine for every dense contraction on the path:
//   conv2d_gradfix.conv2d / conv_transpose2d          (torch_utils/ops/conv2d_gradfix.py:37-45; modulated convolutions of
//                                                      model/generator_sres.py:63-65, discriminator convs of conv2d_resample.py:29-41)
//   F.conv3d of the low-res networks                  (model/generator_lres.py:119,578, model/discriminator_lres.py:172)
//   F.conv1d of the low-res discriminator epilogue    (model/discriminator_lres.py:108-127)
// fp16 tensors run fp16 x fp16 -> fp32; fp32 tensors (the reference keeps TF32 off, train_lres.py:269) are split into
// bf16 hi + lo halves and accumulate hi*hi + lo*hi + hi*lo in fp32 (relative error ~2^-16, three tensor-core products
// instead of one SIMT fp32 pass).
//
// Data layout. Activations are first re-tiled (conv_pack_act_kernel, one streaming pass) from NC(T)HW to channel blocks
// of 8:   X8[instance][block][t][h][w][8]   (16 bytes per pixel and block; instance = sample x group).
// In this layout
//   * a TMA tensor map (8, W, H, T, instance*block) addresses any halo tile with hardware zero fill -- no alignment
//     constraints from odd row pitches (the fp16 NCHW rows of the super-res layers are 4 mod 8 elements long);
//   * the tile lands in shared memory as [block][row][pixel][16 B], which IS the canonical K-major no-swizzle operand
//     layout with the pixel index running linearly at 16 bytes: a filter tap (ky, kx) is nothing but a descriptor start
//     address advanced by (ky * tile_width + kx) * 16 bytes. No shifted copies, no register staging.
//   * N of one MMA runs linearly over the tile INCLUDING its halo columns; the accumulator columns that straddle two rows
//     are computed and dropped in the epilogue (kw - 1 of every tile_width columns).
// GEMM view per instance:  D[co][pix] = sum_{kt} sum_{ci} sum_{ky,kx} W[co][ci][kt][ky][kx] * X[ci][t + kt][y + ky][x + kx]
//   M = 128 output channels (two warpgroups of 64), N = TH x (WT + kw - 1) pixels (<= 256 register columns),
//   K = 16 channels per MMA; the K loop runs over (kt, 16-channel step), every stage issues kh*kw MMAs (one per tap).
//   GEMMs with M <= 64 run in 64-row mode: M = 64, and the two warpgroups split the N columns.
// Weights are re-tiled per call into 128 x 16 (64-row mode: 64 x 16) K-major images per (m-tile, k-step, tap)
// (conv_pack_w_kernel) and arrive with one cp.async.bulk per stage.
//
// Roles (384 threads): warp 0 = TMA producer (one lane), warpgroups 1-2 = wgmma consumers, each with its 64 accumulator rows
// in registers and its own epilogue ([bias, lrelu, gain, clamp] -> NC(T)HW global). Stages hand over through full/empty mbarriers.
//
// Host side (conv_engine.cuh): a call is a ConvShape; fprop_job / dgrad_job derive the forward kernel's job from it,
// plan_igemm tiles a job (host arithmetic only: lvg_convnd_plan reports it) and run_igemm re-tiles and launches; run_wgrad
// runs the weight gradient; backward_dgrad / backward_wgrad run both gradients of a call, sharing one re-tiling of dy where
// the tiles agree. Every workspace is carved from a rooms struct whose total the size queries return. The fused ops that
// drive the engine live in modconv.cu, sres_layer.cu and sres_dblock.cu.

#include <algorithm>
#include <cuda.h>
#include <stdlib.h>
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"
#include "conv_engine.cuh"

namespace lvg {
// conv_pointwise.cu: streaming fp32 kernels for 1x1x1 convolutions with few channels (HBM-bound; the engine would re-tile and pad)
bool pw_supported(int dtype, int groups, int cin, int cout, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, int64_t P);
int pw_conv(const float* x, const float* w, float* y, int n, int cin, int cout, int64_t P, int64_t w_sco, int64_t w_sci, cudaStream_t s);
// conv_pw_tc.cu: every other 1x1x1 forward / input gradient on wgmma, straight from the NC(T)HW tensors (no re-tiling)
bool pw_tc_supported(int dtype, int groups, int cin, int cout, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, int64_t P);
int pw_tc_conv(const void* x, const void* w, void* y, int dtype, int n, int ck, int cm, int64_t P, int64_t w_sm, int64_t w_sk, void* workspace,
               int64_t workspace_bytes, cudaStream_t s, const void* res = nullptr, float rscale = 1.f);
int64_t pw_tc_workspace(int dtype, int ck, int cm);
}

namespace lvg {
namespace {

using namespace tc;

constexpr int kBM = 128;
constexpr int kATile = kBM * 16 * 2;          // one 128 x 16 weight image: 4096 bytes (64-row mode: 2048)
constexpr int kIgemmThreads = 384;           // both kernels: a producer warpgroup and two consumer warpgroups
constexpr int kWidths = 16;                  // conv_igemm_kernel: MMA widths 16, 32, ..., 256 columns
constexpr int kMaxStages = 6;
constexpr int kBSlack = 1024;                // shared memory behind an activation stage that MMAs may read

// Unsigned division of n < 2^31 by a launch constant d >= 1 as a multiply-high and a shift (Granlund and Montgomery):
// mul = ceil(2^(31 + ceil(log2 d)) / d); d = 1 takes mul = 0 and returns n.
struct FastDiv {
    uint32_t d, mul, shift;
};
inline FastDiv fast_div(int d)
{
    FastDiv f = {(uint32_t)d, 0u, 0u};
    int l = 0;
    while ((1ull << l) < (uint64_t)d) l++;
    if (d > 1) { f.mul = (uint32_t)(((1ull << (31 + l)) + d - 1) / d); f.shift = (uint32_t)(l - 1); }
    return f;
}
__device__ __forceinline__ int div_of(int n, const FastDiv& f) { return f.mul ? (int)(__umulhi((uint32_t)n, f.mul) >> f.shift) : n; }

struct IgemmParams {
    const unsigned char* wp;     // packed weights [wgroups][mt][kc][taps_all][a_img]
    void* y;
    const float* bias;           // per output channel (group-local index g*cout + co), or nullptr
    int act;                     // 0 = none, 1 = (x + b) * gain clamped, 2 = lrelu(x + b, alpha) * gain clamped
    float alpha, gain, clamp;    // clamp < 0: none
    int bf16;                    // operands are bf16 (split fp32) instead of fp16; y is fp32 then, fp16 otherwise
    int wgroups, cout, mt, kc;   // kc = 16-channel steps of the packed K axis
    int nblk;                    // channel blocks per instance in X8
    int nimg;                    // operand images per k-step: 1 (fp16) or 2 (split: hi and lo halves of both operands)
    int lo_blk;                  // split: block offset of the lo halves inside an instance of X8
    int to, ho, wo;              // output extent
    int kt, kh, kw, pad_t, pad_h, pad_w;
    int tt, th, wt, wtb, thb;    // tile frames / rows / cols, box cols / rows
    int frame_px;                // thb * wtb: accumulator columns from one frame of the tile to the next
    int ncols;                   // accumulator columns of the tile (multiple of 16, <= 256)
    int m64;                     // 64-row mode (cout <= 64): 64-row weight images, both consumers read the same A and split the columns
    int ncw;                     // MMA width of a consumer: ncols, or in 64-row mode ncols / 2 rounded up to 16
    int a_img;                   // bytes of one weight image: 4096 (128 rows), 2048 (64 rows)
    int tiles_x, tiles_y, tiles_t;
    int64_t total_tiles;         // tiles_x * tiles_y * tiles_t * mt * instances (< 2^31)
    FastDiv div_x, div_y, div_t, div_mt, div_groups;     // tiles_x, tiles_y, tiles_t, mt, wgroups
    int ks;                      // k-steps per stage (> 1 only when kt == 1)
    int stages;
    int a_resident;              // the ring length is a multiple of the stages per tile and every tile of the launch uses the same weights:
                                 // slot s always holds the same weight images -- they are fetched for the first `stages` iterations only
    int a_stage, b_step, b_bytes, b_box, stage_bytes;    // bytes: A per stage, B stride per k-step / per pair of blocks, TMA payload of a pair, whole stage
    int64_t y_cs;                // output channel stride (= to*hos*wos)
    int ostride, hos, wos;       // output decimation (strided convolution): only rows / columns divisible by ostride are stored
    int ths, wts;                // th / ostride, wt / ostride: a row / column tile's origin on the stored grid (tile origins lie on the lattice)
    int pair_store;              // adjacent even / odd accumulator columns are adjacent output elements and y is aligned for
                                 // one 8-byte fp32 / 4-byte half2 store per pair (plan_pairs_columns and an aligned y)
    const float* out_scale;      // per-(instance, output channel, output frame) factor [inst][cout][to] on the accumulator, or nullptr
};

// ------------------------------------------------------------------------------------------------ re-tiling passes


// NC(T)HW -> X8. One thread = one pixel of one channel block: 8 strided reads (coalesced across the warp), one or two
// 16-byte writes. SPLIT: fp32 in, bf16 hi blocks [0, cblk) and lo blocks [cblk, 2 cblk) out.
// Dilation (gradients of strided convolutions): input pixel (t, i, j) of an ih x iw image lands at (t, i*dil, j*dil) of
// the oh x ow output image, which the caller has zeroed.
// `scale` (modulated convolutions): every element is multiplied by scale[instance][channel][frame] in fp32 before it is
// rounded to fp16 / split into bf16 halves; nullptr = the elements are copied as they are.
// GATE (gradients of a layer with bias_act in its epilogue): x is the gradient dy of the layer's output `gy` (same layout,
// stride 1), and every element is first multiplied by G(gy), bias_act's gradient rule (ActGate), in fp32.
struct PackGeom { int64_t thw_in, thw_out; int ih, iw, oh, ow, dil; const float* scale; const void* gy; int act; float alpha, gain, inv_gain, clamp; };

// dy * G(y) as bias_act_elem (bias_act.cu) computes it for grad 1: (dy or dy * alpha by the sign of y / gain) * gain, 0
// where the forward clamped
__device__ __forceinline__ float act_gate(float dy, float yv, const PackGeom& gm)
{
    float v = (gm.act == 2 && !(yv * gm.inv_gain > 0.f)) ? dy * gm.alpha : dy;
    v *= gm.gain;
    return (gm.clamp >= 0.f && !(yv > -gm.clamp && yv < gm.clamp)) ? 0.f : v;
}

template <class TIn, bool SPLIT, bool SCALE, bool GATE>
__device__ __forceinline__ void pack_act_grid(const TIn* __restrict__ x, uint4* __restrict__ y, int64_t inst, int c, int cblk, const PackGeom& gm)
{
    const int64_t thw = gm.thw_in;
    const int64_t total = inst * cblk * thw;
    const int nblk = SPLIT ? 2 * cblk : cblk;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = i % thw;
        const int64_t r = i / thw;
        const int blk = (int)(r % cblk);
        const int64_t in = r / cblk;
        const int c0 = blk * 8;
        const TIn* src = x + ((int64_t)in * c + c0) * thw + p;
        const float* sc = nullptr;           // this pixel's factor of channel c0 (channel stride: frames)
        int64_t frames = 1;
        if constexpr (SCALE) {
            const int64_t hw = (int64_t)gm.ih * gm.iw;
            frames = thw / hw;
            sc = gm.scale + ((int64_t)in * c + c0) * frames + p / hw;
        }
        int64_t po = p;
        if (gm.dil > 1) {
            const int j = (int)(p % gm.iw);
            const int64_t q = p / gm.iw;
            const int ii = (int)(q % gm.ih);
            const int64_t t = q / gm.ih;
            po = (t * gm.oh + (int64_t)ii * gm.dil) * gm.ow + (int64_t)j * gm.dil;
        }
        if constexpr (!SPLIT) {
            alignas(16) unsigned short v[8];
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = (c0 + j < c) ? __half_as_ushort(__ldg(reinterpret_cast<const __half*>(src) + (int64_t)j * thw)) : (unsigned short)0;
            if constexpr (GATE) {
                const __half* gy = reinterpret_cast<const __half*>(gm.gy) + ((int64_t)in * c + c0) * thw + p;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (c0 + j < c)
                        v[j] = __half_as_ushort(__float2half_rn(act_gate(__half2float(__ushort_as_half(v[j])), __half2float(__ldg(gy + (int64_t)j * thw)), gm)
                                                                * __ldg(sc + j * frames)));
            } else if constexpr (SCALE) {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (c0 + j < c) v[j] = __half_as_ushort(__float2half_rn(__half2float(__ushort_as_half(v[j])) * __ldg(sc + j * frames)));
            }
            y[((int64_t)in * nblk + blk) * gm.thw_out + po] = *reinterpret_cast<const uint4*>(v);
        } else {
            alignas(16) unsigned short hi[8], lo[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                float f = (c0 + j < c) ? __ldg(reinterpret_cast<const float*>(src) + (int64_t)j * thw) : 0.f;
                if constexpr (GATE) {
                    if (c0 + j < c)
                        f = act_gate(f, __ldg(reinterpret_cast<const float*>(gm.gy) + ((int64_t)in * c + c0 + j) * thw + p), gm) * __ldg(sc + j * frames);
                } else if constexpr (SCALE) {
                    if (c0 + j < c) f *= __ldg(sc + j * frames);
                }
                hi[j] = bf16_bits(f);
                lo[j] = bf16_bits(f - bf16_val(hi[j]));
            }
            y[((int64_t)in * nblk + blk) * gm.thw_out + po] = *reinterpret_cast<const uint4*>(hi);
            y[((int64_t)in * nblk + cblk + blk) * gm.thw_out + po] = *reinterpret_cast<const uint4*>(lo);
        }
    }
}

template <class TIn, bool SPLIT, bool SCALE>
__global__ void __launch_bounds__(256) conv_pack_act_kernel(const TIn* __restrict__ x, uint4* __restrict__ y, int64_t inst, int c,
                                                             int cblk, PackGeom gm)
{
    pack_act_grid<TIn, SPLIT, SCALE, false>(x, y, inst, c, cblk, gm);
}

// the re-tiling of a gradient dy times bias_act's gradient rule G(gy) and the factor
template <class TIn, bool SPLIT>
__global__ void __launch_bounds__(256) conv_pack_grad_kernel(const TIn* __restrict__ x, uint4* __restrict__ y, int64_t inst, int c,
                                                              int cblk, PackGeom gm)
{
    pack_act_grid<TIn, SPLIT, true, true>(x, y, inst, c, cblk, gm);
}

// launches the re-tiling of one activation tensor (zeroing the target first when it is dilated)
// (gate: the scaled re-tiling of a gradient times bias_act's gradient rule; it needs a scale and unit dilation)
int pack_act(const void* x, void* x8, int split, int64_t inst, int c, int cblk, int t, int ih, int iw, int oh, int ow, int dil, cudaStream_t s,
             const float* scale = nullptr, const ActGate* gate = nullptr)
{
    PackGeom gm = {};
    gm.thw_in = (int64_t)t * ih * iw; gm.thw_out = (int64_t)t * oh * ow; gm.ih = ih; gm.iw = iw; gm.oh = oh; gm.ow = ow; gm.dil = dil;
    gm.scale = scale;
    const bool gated = gate != nullptr && gate->y != nullptr;
    if (gated) {
        LVG_REQUIRE(scale != nullptr && dil == 1 && (gate->act == 1 || gate->act == 2), "convnd: a gated re-tiling needs a scale, unit stride and linear / lrelu");
        gm.gy = gate->y; gm.act = gate->act; gm.alpha = gate->alpha; gm.gain = gate->gain; gm.clamp = gate->clamp;
        gm.inv_gain = gate->gain != 0.f ? 1.f / gate->gain : 0.f;
    }
    if (dil > 1) LVG_CUDA(cudaMemsetAsync(x8, 0, (size_t)(inst * (split ? 2 : 1) * cblk * gm.thw_out * 16), s));
    const int64_t total = inst * cblk * gm.thw_in;
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 64;
    if (blocks > cap) blocks = cap;
    // (the scaled variants are separate instantiations: the unscaled re-tiling stays the plain copy it was)
    if (gated && split) conv_pack_grad_kernel<float, true><<<(unsigned)blocks, 256, 0, s>>>((const float*)x, (uint4*)x8, inst, c, cblk, gm);
    else if (gated) conv_pack_grad_kernel<__half, false><<<(unsigned)blocks, 256, 0, s>>>((const __half*)x, (uint4*)x8, inst, c, cblk, gm);
    else if (split && scale) conv_pack_act_kernel<float, true, true><<<(unsigned)blocks, 256, 0, s>>>((const float*)x, (uint4*)x8, inst, c, cblk, gm);
    else if (split) conv_pack_act_kernel<float, true, false><<<(unsigned)blocks, 256, 0, s>>>((const float*)x, (uint4*)x8, inst, c, cblk, gm);
    else if (scale) conv_pack_act_kernel<__half, false, true><<<(unsigned)blocks, 256, 0, s>>>((const __half*)x, (uint4*)x8, inst, c, cblk, gm);
    else conv_pack_act_kernel<__half, false, false><<<(unsigned)blocks, 256, 0, s>>>((const __half*)x, (uint4*)x8, inst, c, cblk, gm);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}


// weights -> tile images.  Element (m, k, tap) of the logical A matrix of group g sits at
//   w[g * gstride + m * sm + k * sk + (flip ? taps-1-tap : tap)]
// fprop: m = co, k = ci (sm = cin*taps, sk = taps); dgrad: m = ci, k = co (sm = taps, sk = cin*taps), taps mirrored.
// Image of one 128 x 16 tile (K-major, no swizzle): byte offset(m, k) = (k/8)*2048 + (m/8)*128 + (m%8)*16 + (k%8)*2.
// SPLIT: every (k-step, tap) gets TWO images, the bf16 hi and lo halves of the fp32 weights; the main loop pairs them with
// the hi / lo activation blocks: hi*hi + hi*lo + lo*hi (each operand half is fetched once per k-step).
// One CTA = one (group, m-tile, k-step). The 128 x 16 x taps source elements form contiguous RUNS in memory (fprop: one
// run of 16*taps elements per output channel; dgrad: one run of 128*taps elements per k): a warp copies a run into shared
// memory with aligned 4-byte loads (no per-element index arithmetic), then every thread assembles one 16-byte image row
// from 8 shared-memory reads and consecutive threads write consecutive rows (512 contiguous bytes per warp).
// 64-row mode (GEMMs with at most 64 rows): 64 x 16 images of 2048 bytes, byte offset(m, k) = (k/8)*1024 + (m/8)*128 +
// (m%8)*16 + (k%8)*2, row = channel; both consumer warpgroups read the whole image.
// Rows of the 128-row weight image (= accumulator rows). An m-tile with fewer than 128 output channels spreads them evenly
// over the four 32-row quarters (`per` channels at the start of each) instead of filling quarter after quarter, so that
// both consumer warpgroups and all their warps share the epilogue's store work of a 32- or 64-channel layer. Channels
// >= 4 * per (zero rows) take the remaining rows in order.
__host__ __device__ __forceinline__ int m_rows_per_quadrant(int channels_left)
{
    const int cv = channels_left < kBM ? (channels_left > 0 ? channels_left : 0) : kBM;
    return cv >= kBM ? 32 : (cv + 3) / 4 > 0 ? (cv + 3) / 4 : 1;
}
__host__ __device__ __forceinline__ int m_row_of_channel(int ch, int per)
{
    if (per >= 32) return ch;
    if (ch < 4 * per) return (ch / per) * 32 + ch % per;
    const int r = ch - 4 * per;
    return (r / (32 - per)) * 32 + per + r % (32 - per);
}

// inverse of m_row_of_channel: the channel (relative to the m-tile) held by image row `row`
__host__ __device__ __forceinline__ int m_channel_of_row(int row, int per)
{
    if (per >= 32) return row;
    const int q = row / 32, i = row % 32;
    return i < per ? q * per + i : 4 * per + q * (32 - per) + (i - per);
}

template <class TIn, bool SPLIT>
__global__ void __launch_bounds__(256) conv_pack_w_kernel(const TIn* __restrict__ w, unsigned char* __restrict__ wp, int m_total, int k_total,
                                                           int kpad, int taps, int64_t gstride, int64_t sm, int64_t sk, int flip, int mt, int kc,
                                                           int rows_per_pass, int rows_per_cta, int img_rows)
{
    extern __shared__ uint32_t sw32[];               // [runs][pitch] words, then the runs' element offsets
    constexpr int ES = (int)sizeof(TIn);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int kci = blockIdx.x % kc;
    const int mti = (blockIdx.x / kc) % mt;
    const int g = blockIdx.x / (kc * mt);
    const int k0 = kci * 16;
    (void)kpad;
    constexpr int NIMG = SPLIT ? 2 : 1;
    const TIn* wg = w + (int64_t)g * gstride;
    const bool mrows = sk < sm;                      // fprop layout: runs along (k, tap) per m; else runs along (m, tap) per k
    const int R = rows_per_pass;
    const int run_el = mrows ? 16 * taps : R * taps;
    const int pitch = ((run_el * ES + 2 + 3) / 4) | 1;
    const int max_runs = mrows ? R : 16;
    int* s_off = reinterpret_cast<int*>(sw32 + (size_t)max_runs * pitch);
    const int img = img_rows * 32;                   // bytes of one image
    unsigned char* dst0 = wp + ((((int64_t)g * mt + mti) * kc + kci) * taps) * (int64_t)(NIMG * img);
    const int kvalid = max(0, min(16, k_total - k0));
    const int per = m_rows_per_quadrant(m_total - mti * kBM);
    // blockIdx.y = chunk of rows_per_cta image rows (small layers have only a handful of (group, m-tile, k-step) blocks: the
    // row chunks spread their latency-bound staging over more SMs)
    const int row_end = min(img_rows, ((int)blockIdx.y + 1) * rows_per_cta);
    for (int r0 = (int)blockIdx.y * rows_per_cta; r0 < row_end; r0 += R) {
        const int Rn = min(R, row_end - r0);
        const int m0 = mti * img_rows + r0;
        const int mvalid = max(0, min(Rn, m_total - m0));
        const int len = mrows ? kvalid * taps : mvalid * taps;             // valid elements of a run
        const int nruns = len > 0 ? (mrows ? mvalid : kvalid) : 0;
        for (int run = warp; run < nruns; run += 8) {
            const int64_t e0 = mrows ? (int64_t)(m0 + run) * sm + (int64_t)k0 * sk : (int64_t)(k0 + run) * sk + (int64_t)m0 * sm;
            const unsigned char* gb = reinterpret_cast<const unsigned char*>(wg + e0);
            const int a = (int)(reinterpret_cast<uintptr_t>(gb) & 3);       // 0, or 2 for an odd fp16 element offset
            const uint32_t* gw = reinterpret_cast<const uint32_t*>(gb - a);
            const int nbytes = len * ES + a;
            const int nwords = (nbytes + 3) / 4;
            // whole words strictly inside the run: four independent loads in flight per lane
            const int w_lo = a != 0 ? 1 : 0, w_hi = (nbytes & 3) != 0 ? nwords - 1 : nwords;
            int wi = w_lo + lane;
            for (; wi + 96 < w_hi; wi += 128) {
                const uint32_t v0 = __ldg(gw + wi), v1 = __ldg(gw + wi + 32), v2 = __ldg(gw + wi + 64), v3 = __ldg(gw + wi + 96);
                uint32_t* d = sw32 + run * pitch + wi;
                d[0] = v0; d[32] = v1; d[64] = v2; d[96] = v3;
            }
            for (; wi < w_hi; wi += 32) sw32[run * pitch + wi] = __ldg(gw + wi);
            if (lane == 0 && a != 0) sw32[run * pitch] = (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(gb)) << 16;              // do not touch bytes before the run
            if (lane == 1 && w_hi < nwords && !(a != 0 && nwords == 1))
                sw32[run * pitch + nwords - 1] = (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(gw + nwords - 1));              // ... or after it
            if (lane == 0) s_off[run] = a / ES;
        }
        __syncthreads();
        const bool pow2 = Rn == kBM;
        for (int o = threadIdx.x; o < taps * 2 * Rn; o += 256) {
            int mrow, k8, tap;
            if (pow2) { mrow = o & (kBM - 1); k8 = (o >> 7) & 1; tap = o >> 8; }
            else { mrow = o % Rn; k8 = (o / Rn) % 2; tap = o / (2 * Rn); }
            const int wtap = flip ? taps - 1 - tap : tap;
            alignas(16) unsigned short v[8], vlo[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int k = k8 * 8 + j;
                const int run = mrows ? mrow : k;
                const int idx = mrows ? k * taps + wtap : mrow * taps + wtap;
                float f = 0.f;
                unsigned short hbits = 0;
                if (mrow < mvalid && k < kvalid) {
                    if constexpr (ES == 2) hbits = reinterpret_cast<const unsigned short*>(sw32 + run * pitch)[s_off[run] + idx];
                    else f = __uint_as_float(sw32[run * pitch + idx]);
                }
                if constexpr (SPLIT) {
                    if constexpr (ES == 2) f = __half2float(__ushort_as_half(hbits));
                    const unsigned short h = bf16_bits(f);
                    v[j] = h;
                    vlo[j] = bf16_bits(f - bf16_val(h));
                } else {
                    v[j] = ES == 2 ? hbits : __half_as_ushort(__float2half_rn(f));
                }
            }
            const int row = img_rows == kBM ? m_row_of_channel(r0 + mrow, per) : r0 + mrow;
            unsigned char* dimg = dst0 + (size_t)tap * (NIMG * img) + k8 * (img / 2) + row * 16;
            *reinterpret_cast<uint4*>(dimg) = *reinterpret_cast<const uint4*>(v);
            if constexpr (SPLIT) *reinterpret_cast<uint4*>(dimg + img) = *reinterpret_cast<const uint4*>(vlo);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ main kernel

__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
                 : "memory");
}

// X8 seen as 8-byte elements: (2*W, H, T, instance*block). A pixel of a block is two elements, so a box row is one
// contiguous run of 16*width bytes (with a 16-byte innermost dimension TMA moves one pixel per request).
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
                 : "memory");
}

struct TileCoord { int ox0, oy0, t0, mti, inst, grp, ix, iy; };

__device__ __forceinline__ TileCoord decode_tile(const IgemmParams& p, int L)
{
    TileCoord c;
    int q = div_of(L, p.div_x);
    c.ix = L - q * p.tiles_x;
    int r = div_of(q, p.div_y);
    c.iy = q - r * p.tiles_y;
    q = div_of(r, p.div_t);
    c.t0 = (r - q * p.tiles_t) * p.tt;
    c.inst = div_of(q, p.div_mt);
    c.mti = q - c.inst * p.mt;
    c.grp = c.inst - div_of(c.inst, p.div_groups) * p.wgroups;
    c.ox0 = c.ix * p.wt; c.oy0 = c.iy * p.th;
    return c;
}

// Column map of the epilogue. Which output element an accumulator column holds depends on the launch only: column n is
// (frame f, row r, col cc) of the tile, stored at f * hos * wos + (r / ostride) * wos + cc / ostride past the tile's
// origin on the stored grid, unless it is a halo column, lies off the stride lattice or is past ncols. Each CTA builds the
// map once; a tile then needs only its origin and its clipped extents, and the epilogue does no division.
// The clip test is one subtraction: key = cc | r << 11 | f << 22 (10-, 10- and 8-bit fields), a tile's limit word holds
// (extent - 1) of each axis in the same fields with the guard bits 10, 21 and 30 set; (limit - key) keeps a field's guard
// bit exactly when key's field is within the extent (no borrow crosses a guard). Columns never stored get a key whose cc
// field (1023) no tile accepts.
constexpr uint32_t kKeyGuards = (1u << 10) | (1u << 21) | (1u << 30);
constexpr uint32_t kKeyNever = 1023u;
constexpr int kMapCols = 256;                // at most 256 accumulator columns per tile (both halves in 64-row mode)

__device__ __forceinline__ uint32_t col_limit(int tl, int hl, int wl)
{
    return ((uint32_t)(wl - 1) | (uint32_t)(hl - 1) << 11 | (uint32_t)(tl - 1) << 22) | kKeyGuards;
}
__device__ __forceinline__ bool col_in_tile(uint32_t key, uint32_t limit) { return ((limit - key) & kKeyGuards) == kKeyGuards; }

// [bias, lrelu, gain, clamp] as the reference applies them (act 0: the accumulator as it is)
__device__ __forceinline__ float epilogue_value(const IgemmParams& p, float v, float bias)
{
    if (p.act) {
        v += bias;
        if (p.act == 2) v = v < 0.f ? v * p.alpha : v;
        v *= p.gain;
        if (p.clamp >= 0.f) v = fminf(fmaxf(v, -p.clamp), p.clamp);
    }
    return v;
}

// Persistent: CTA b works on tiles b, b + gridDim.x, ... (pixel tile fastest, so that concurrently running CTAs share the
// weight tiles of one (instance, m-tile) in L2). The operand ring runs across tile boundaries, so the producer fetches the
// first stages of tile i + 1 while the consumers store tile i.
// Roles (384 threads): warp 0 = TMA producer (one lane); warpgroups 1 and 2 = MMA + epilogue for accumulator rows 0-63 and
// 64-127 of the weight images, each over all ncols columns (NW = ncols). 64-row mode (at most 64 output rows): both read
// the same 64-row images, warpgroup 1 takes columns [0, NW), warpgroup 2 [NW, 2 NW) (NW = ncols / 2 rounded up to 16;
// columns >= ncols are computed and dropped). Each consumer holds its 64 x NW fp32 accumulator in registers, issues one
// m64nNWk16 per tap and product, and releases a stage once the wgmma group that read it has completed.
template <bool BF16, int NW, bool OSCALE>
__global__ void __launch_bounds__(kIgemmThreads, 1) conv_igemm_kernel(const __grid_constant__ CUtensorMap tmx, const IgemmParams p)
{
    using OutT = typename std::conditional<BF16, float, __half>::type;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
    __shared__ __align__(16) int2 col_map[kMapCols];         // accumulator column -> (offset past the tile origin, clip key)
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);

    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);     // warpgroup index, warp-uniform to the compiler
    const int taps2 = p.kh * p.kw;
    const int kchunks = (p.kc + p.ks - 1) / p.ks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    for (int n = threadIdx.x; n < (p.m64 ? 2 * NW : NW); n += kIgemmThreads) {
        const int f = n / p.frame_px, rem = n - f * p.frame_px;
        const int r = rem / p.wtb, cc = rem - r * p.wtb;
        const bool st = n < p.ncols && f < p.tt && r < p.th && cc < p.wt && r % p.ostride == 0 && cc % p.ostride == 0;
        col_map[n] = st ? make_int2((f * p.hos + r / p.ostride) * p.wos + cc / p.ostride, (int)((uint32_t)cc | (uint32_t)r << 11 | (uint32_t)f << 22))
                        : make_int2(0, (int)kKeyNever);
    }
    __syncthreads();

    if (wg == 0) {
        if (warp == 0 && elect_one()) {
            int it = 0, s = 0;
            uint32_t phase = 0;                               // (it / stages) & 1: the ring position kept without a division
            for (int L = blockIdx.x; L < p.total_tiles; L += gridDim.x) {
                const TileCoord c = decode_tile(p, L);
                const unsigned char* wpg = p.wp + (((int64_t)c.grp * p.mt + c.mti) * p.kc) * (int64_t)(p.kt * taps2) * (p.nimg * p.a_img);
                const int blk0 = c.inst * p.nblk;
                for (int kt = 0; kt < p.kt; kt++) {
                    for (int kcix = 0; kcix < kchunks; kcix++, it++, s = s + 1 == p.stages ? (phase ^= 1u, 0) : s + 1) {
                        if (it >= p.stages) mbar_wait(&empty_bar[s], phase ^ 1u);
                        unsigned char* st = smem + (size_t)s * p.stage_bytes;
                        const int k0 = kcix * p.ks;
                        const int nks = min(p.ks, p.kc - k0);
                        const bool load_a = !p.a_resident || it < p.stages;
                        const uint32_t a_bytes = load_a ? (uint32_t)(nks * taps2 * p.nimg * p.a_img) : 0u;
                        mbar_expect_tx(&full_bar[s], a_bytes + (uint32_t)(nks * p.nimg * p.b_box));
                        // A: kt == 1 -> the nks steps' tiles are contiguous; kt > 1 -> ks == 1, the taps of this kt are contiguous
                        if (load_a) bulk_copy_g2s(st, wpg + ((int64_t)k0 * p.kt + kt) * (int64_t)taps2 * (p.nimg * p.a_img), a_bytes, &full_bar[s]);
                        for (int j = 0; j < nks; j++) {
                            const int kb = (k0 + j) * 2;
                            for (int im = 0; im < p.nimg; im++)
                                tma_load_4d(st + p.a_stage + (size_t)j * p.b_step + (size_t)im * p.b_bytes, &tmx, 2 * (c.ox0 - p.pad_w), c.oy0 - p.pad_h,
                                            c.t0 + kt - p.pad_t, blk0 + im * p.lo_blk + kb, &full_bar[s]);
                        }
                    }
                }
            }
        }
    } else if (wg >= 1) {
        const int cw = wg - 1;
        const int tid = threadIdx.x % 128, wq = tid / 32;
        const uint32_t blk_bytes = (uint32_t)p.b_box / 2;
        const uint32_t a_hi = desc_hi(128), b_hi = desc_hi(128);
        const uint32_t a_tap = (uint32_t)(p.nimg * p.a_img) >> 4, a_lo_img = (uint32_t)p.a_img >> 4, b_lo_img = (uint32_t)p.b_bytes >> 4;
        // 128-row images: this warpgroup's 64 rows start 1024 bytes into an image; 64-row mode: its columns start NW pixels in
        const uint32_t a_row0 = p.m64 ? 0u : (uint32_t)cw * 1024u;
        const int col0 = p.m64 ? cw * NW : 0;
        int s = 0;
        uint32_t phase = 0;
        for (int L = blockIdx.x; L < p.total_tiles; L += gridDim.x) {
            const TileCoord c = decode_tile(p, L);
            float acc[NW / 2];
#pragma unroll
            for (int i = 0; i < NW / 2; i++) acc[i] = 0.f;
            int prev = -1;
            for (int kt = 0; kt < p.kt; kt++) {
                for (int kcix = 0; kcix < kchunks; kcix++, s = s + 1 == p.stages ? (phase ^= 1u, 0) : s + 1) {
                    mbar_wait(&full_bar[s], phase);
                    wgmma_fence();
                    const uint32_t st = smem_u32(smem + (size_t)s * p.stage_bytes);
                    const int nks = min(p.ks, p.kc - kcix * p.ks);
                    // descriptors as (lo, hi) words, stepped with 32-bit adds on the low word (address >> 4): the next tap's weight
                    // image(s) + nimg * a_img bytes, the next tap column + 16 bytes, the next tap row + wtb * 16 bytes, the next
                    // accumulator column + 16 bytes. A's LBO (the second 8-channel half) is half an image.
                    for (int j = 0; j < nks; j++) {
                        uint32_t a_lo = desc_lo(st + (uint32_t)(j * taps2 * p.nimg * p.a_img) + a_row0, (uint32_t)p.a_img / 2);
                        const uint32_t b_base = desc_lo(st + (uint32_t)p.a_stage + (uint32_t)j * (uint32_t)p.b_step, blk_bytes) + (uint32_t)col0;
                        for (int ky = 0; ky < p.kh; ky++) {
                            for (int kx = 0; kx < p.kw; kx++, a_lo += a_tap) {
                                const uint32_t b_lo = b_base + (uint32_t)(ky * p.wtb + kx);
                                // fp16: one product; split: hi*hi, hi*lo, lo*hi (A image hi, hi, lo; B image hi, lo, hi)
                                wgmma_m64nNk16<BF16, NW, 0, 0>(acc, a_lo, a_hi, b_lo, b_hi);
                                if constexpr (BF16) {
                                    wgmma_m64nNk16<BF16, NW, 0, 0>(acc, a_lo, a_hi, b_lo + b_lo_img, b_hi);
                                    wgmma_m64nNk16<BF16, NW, 0, 0>(acc, a_lo + a_lo_img, a_hi, b_lo, b_hi);
                                }
                            }
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                          // the group of the previous stage has completed: release its slot
                    mbar_arrive_if(&empty_bar[prev >= 0 ? prev : 0], prev >= 0 && tid == 0);
                    prev = s;
                }
            }
            wgmma_wait<0>();
            mbar_arrive_if(&empty_bar[prev], tid == 0);

            // ---- epilogue: registers -> [bias, lrelu, gain, clamp] -> NC(T)HW global. This thread holds accumulator rows
            // r and r + 8 (conv_pack_w_kernel's row order -> channel) and column pairs col0 + 8 j + 2 (lane % 4); the column
            // map gives each column's place past the tile origin.
            const int per = m_rows_per_quadrant(p.cout - c.mti * kBM);
            const uint32_t limit = col_limit(min(p.tt, p.to - c.t0), min(p.th, p.ho - c.oy0), min(p.wt, p.wo - c.ox0));
            const int64_t tile_off = ((int64_t)c.t0 * p.hos + c.iy * p.ths) * p.wos + c.ix * p.wts;
            OutT* yrow[2];
            float bias[2];
            bool rok[2];
            const float* osc[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row = wq * 16 + lane / 4 + 8 * h;
                const int ch = p.m64 ? row : m_channel_of_row(cw * 64 + row, per);
                const int co = c.mti * kBM + ch;
                rok[h] = ch < kBM && co < p.cout;
                bias[h] = (p.bias != nullptr && rok[h]) ? __ldg(p.bias + (int64_t)c.grp * p.cout + co) : 0.f;
                yrow[h] = reinterpret_cast<OutT*>(p.y) + ((int64_t)c.inst * p.cout + co) * p.y_cs + tile_off;
                osc[h] = OSCALE ? p.out_scale + ((int64_t)c.inst * p.cout + co) * p.to + c.t0 : nullptr;
            }
            const int2* cmap = col_map + col0 + 2 * (lane % 4);
            if (p.pair_store) {
                // columns 2i and 2i + 1 are stored together or not at all, at adjacent addresses
#pragma unroll
                for (int j = 0; j < NW / 8; j++) {
                    const int2 m = cmap[j * 8];
                    if (!col_in_tile((uint32_t)m.y, limit)) continue;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        if (!rok[h]) continue;
                        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                        if constexpr (OSCALE) { const float s = __ldg(osc[h] + ((uint32_t)m.y >> 22)); v0 *= s; v1 *= s; }
                        v0 = epilogue_value(p, v0, bias[h]);
                        v1 = epilogue_value(p, v1, bias[h]);
                        if constexpr (BF16) *reinterpret_cast<float2*>(yrow[h] + m.x) = make_float2(v0, v1);
                        else *reinterpret_cast<__half2*>(yrow[h] + m.x) = __floats2half2_rn(v0, v1);
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < NW / 8; j++) {
                    const int4 m = *reinterpret_cast<const int4*>(cmap + j * 8);
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int off = e ? m.z : m.x;
                        const uint32_t key = (uint32_t)(e ? m.w : m.y);
                        if (!col_in_tile(key, limit)) continue;
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            if (!rok[h]) continue;
                            float v = acc[4 * j + 2 * h + e];
                            if constexpr (OSCALE) v *= __ldg(osc[h] + (key >> 22));
                            v = epilogue_value(p, v, bias[h]);
                            if constexpr (BF16) yrow[h][off] = v;
                            else yrow[h][off] = __float2half_rn(v);
                        }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
        return reinterpret_cast<EncodeTiledFn>(f);
    }();
    return fn;
}

// tensor map over a channel-block-of-8 tensor [blocks][t][h (pitch_hw / pitch_w rows)][w][8 x 2 bytes], seen as 8-byte
// elements: (2 w, h, t, blocks); box = box_w pixels x box_h rows x box_t frames x box_blk blocks
int encode_map(CUtensorMap* tm, void* base, int w, int h, int t, int64_t blocks, int64_t pitch_w, int64_t pitch_hw, int64_t pitch_thw, int box_w,
               int box_h, int box_t, int box_blk)
{
    EncodeTiledFn enc = encode_fn();
    LVG_REQUIRE(enc != nullptr, "convnd: cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dims[4] = {(cuuint64_t)w * 2, (cuuint64_t)h, (cuuint64_t)t, (cuuint64_t)blocks};
    const cuuint64_t strides[3] = {(cuuint64_t)pitch_w * 16, (cuuint64_t)pitch_hw * 16, (cuuint64_t)pitch_thw * 16};
    const cuuint32_t box[4] = {(cuuint32_t)box_w * 2, (cuuint32_t)box_h, (cuuint32_t)box_t, (cuuint32_t)box_blk};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    LVG_REQUIRE(box_w <= 128 && box_h <= 256 && box_t <= 256 && box_blk <= 256, "convnd: TMA box too large");
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LVG_REQUIRE(r == CUDA_SUCCESS, "convnd: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return LVG_OK;
}

inline int env_flag(const char* name, int dflt)
{
    const char* e = getenv(name);
    return e ? atoi(e) : dflt;
}

bool nd_supported(int dtype, int kt, int kh, int kw)
{
    return (dtype == LVG_F16 || dtype == LVG_F32) && kt >= 1 && kh >= 1 && kw >= 1 && kh * kw <= 9 && kt <= 7;
}

Geometry job_geometry(const IgemmJob& j)
{
    return geometry(j.dtype == LVG_F32, (int64_t)j.n * j.groups, j.groups, j.ck, j.cm, (int64_t)j.t * j.h * j.wd, j.kt * j.kh * j.kw);
}

IgemmRooms igemm_rooms_of(const Geometry& g, bool x8_pre) { return {round256(g.w_bytes), x8_pre ? 0 : g.act_bytes}; }

// Accumulator columns 2i and 2i + 1 are the same output row's elements x and x + 1 with x even, both stored or both
// clipped, and every such pair starts at an even element offset: unit stride, even tile and box widths (so even frame
// and row strides in the accumulator), an even output width and channel stride. With a y aligned to a pair's size the
// epilogue stores one 8-byte fp32 / 4-byte half2 per pair.
bool plan_pairs_columns(const IgemmParams& p)
{
    return p.ostride == 1 && p.wt % 2 == 0 && p.wtb % 2 == 0 && p.wo % 2 == 0 && p.y_cs % 2 == 0;
}

// dynamic shared memory of a launch: the stage ring and its 128-byte alignment
int igemm_smem_bytes(const IgemmParams& p) { return p.stages * p.stage_bytes + 128; }

// The tiling of a job: host arithmetic only (no CUDA call, no pointer dereferenced). lvg_convnd_plan hands it out.
int plan_igemm(const IgemmJob& j, IgemmParams& p)
{
    const int kt = j.kt, kh = j.kh, kw = j.kw, ostride = j.ostride;
    const int64_t inst = (int64_t)j.n * j.groups;
    const Geometry g = job_geometry(j);
    LVG_REQUIRE(inst * g.nblk < (1ll << 31), "convnd: too many channel blocks for a tensor map");

    memset(&p, 0, sizeof(p));
    p.y = j.y; p.bias = j.bias; p.act = j.act; p.alpha = j.alpha; p.gain = j.gain; p.clamp = j.clamp; p.out_scale = j.out_scale;
    p.bf16 = j.dtype == LVG_F32 ? 1 : 0;
    p.wgroups = j.groups; p.cout = j.cm; p.mt = g.mt; p.kc = g.kc; p.nblk = g.nblk;
    p.nimg = g.nimg; p.lo_blk = g.cblk;
    p.m64 = g.m64; p.a_img = g.a_img;
    p.to = j.t + 2 * j.pad_t - kt + 1; p.ho = j.h + 2 * j.pad_h - kh + 1; p.wo = j.wd + 2 * j.pad_w - kw + 1;
    LVG_REQUIRE(p.to >= 1 && p.ho >= 1 && p.wo >= 1, "convnd: empty output");
    p.kt = kt; p.kh = kh; p.kw = kw; p.pad_t = j.pad_t; p.pad_h = j.pad_h; p.pad_w = j.pad_w;
    // tile: whole rows (and, for small frames, several frames) up to 256 accumulator columns (the register accumulator of a
    // consumer warpgroup: 128 fp32 registers per thread); wide images are cut into column tiles. LVG_CONV_COLS lowers it.
    const char* cb_env = getenv("LVG_CONV_COLS");
    const int taps2 = kh * kw;
    const int smem_budget = 224 * 1024;
    p.ostride = ostride;
    p.hos = (p.ho - 1) / ostride + 1; p.wos = (p.wo - 1) / ostride + 1;
    p.ks = (kt == 1) ? (taps2 == 1 ? 4 : (taps2 <= 3 ? 2 : 1)) : 1;
    if (p.ks > g.kc) p.ks = g.kc;
    p.a_stage = p.ks * taps2 * g.nimg * g.a_img;
    // the column budget shrinks until two stages fit shared memory (split precision doubles both operands of a stage); column
    // tiles are at most max_wt pixels wide, a TMA box row (256 8-byte elements = 128 pixels) with its kw - 1 halo columns.
    // When no budget fits at that width, narrower column tiles are tried: the row tiles of a strided convolution take at least
    // `ostride` rows each, and tall kernels in split precision need large stages.
    int col_budget0 = cb_env ? atoi(cb_env) : 256;
    if (col_budget0 > 256) col_budget0 = 256;
    bool fits = false;
    for (int max_wt = 128 - (kw - 1); !fits; max_wt -= 8) {
        LVG_REQUIRE(max_wt >= ostride, "convnd: no tile fits shared memory");
        for (int col_budget = col_budget0; col_budget >= 64 && !fits; col_budget -= 64) {
            p.tiles_x = (p.wo + max_wt - 1) / max_wt;
            p.wt = (p.wo + p.tiles_x - 1) / p.tiles_x;
            p.wtb = p.wt + kw - 1;
            p.th = col_budget / p.wtb;
            if (p.th > p.ho) p.th = p.ho;
            if (p.th < 1) p.th = 1;
            p.tiles_y = (p.ho + p.th - 1) / p.th;
            p.th = (p.ho + p.tiles_y - 1) / p.tiles_y;           // balance the row tiles
            if (ostride > 1) {                                     // tile origins on the output lattice, column tiles within max_wt
                if (p.tiles_x > 1) {
                    p.wt = std::min(round_up(p.wt, ostride), max_wt / ostride * ostride);
                    p.wtb = p.wt + kw - 1;
                    p.tiles_x = (p.wo + p.wt - 1) / p.wt;
                    if (p.th * p.wtb > col_budget) p.th = col_budget / p.wtb;
                }
                if (p.th < p.ho) { p.th = p.th / ostride * ostride; if (p.th < ostride) p.th = ostride; }
                p.tiles_y = (p.ho + p.th - 1) / p.th;
            }
            p.thb = p.th + kh - 1;
            p.frame_px = p.thb * p.wtb;
            p.tt = 1;
            if (p.tiles_y == 1 && p.tiles_x == 1) {                // whole frames: take as many as fit
                while (p.tt < p.to && p.tt * p.frame_px + p.th * p.wtb <= col_budget && p.tt < 64) p.tt++;
            }
            p.tiles_t = (p.to + p.tt - 1) / p.tt;
            p.tt = (p.to + p.tiles_t - 1) / p.tiles_t;
            p.ncols = round_up((p.tt - 1) * p.frame_px + p.th * p.wtb, 16);
            // TMA writes the two 8-channel blocks of a k-step densely: block 1 starts tt*thb*wtb*16 bytes after block 0 (= LBO);
            // every pair of blocks starts at a 128-byte multiple (TMA destination alignment)
            p.b_box = 2 * p.tt * p.frame_px * 16;                  // one pair of blocks as TMA writes it
            p.b_bytes = round_up(p.b_box, 128);
            p.b_step = g.nimg * p.b_bytes;
            // + slack: the last taps and (64-row mode) the columns of the second warpgroup past ncols read up to 50 pixels past
            // the tile
            p.stage_bytes = round_up(p.a_stage + p.ks * p.b_step + kBSlack, 128);
            fits = p.ncols <= 256 && 2 * p.stage_bytes <= smem_budget;
        }
    }
    LVG_REQUIRE(p.th >= 1 && p.ncols <= 256 && p.ncols >= 16, "convnd: tile geometry");
    p.ncw = p.m64 ? round_up(p.ncols / 2, 16) : p.ncols;
    p.stages = 2;
    while (p.stages < kMaxStages && (p.stages + 1) * p.stage_bytes <= smem_budget) p.stages++;
    // Short K loops (few input channels, 1x1 / 1x3x3 kernels): when the ring can be cut to a multiple of the stages one tile
    // takes, slot s sees the same (kt, k-chunk) on every tile -- with one weight set for the whole launch (no groups, one
    // m-tile) the weight images stay where the first pass put them and only the activation tiles stream (the weight images
    // of a 32-channel 3x3 layer are 72 KB per k-step against 21 KB of activations: the re-fetch per 256-pixel tile was the
    // L2 -> SM traffic of these layers).
    {
        const int period = kt * ((g.kc + p.ks - 1) / p.ks);
        p.a_resident = 0;
        if (j.groups == 1 && g.mt == 1 && period <= p.stages && env_flag("LVG_CONV_RESIDENT_W", 1)) {
            p.stages = p.stages / period * period;
            p.a_resident = 1;
        }
    }
    p.y_cs = (int64_t)p.to * p.hos * p.wos;
    p.total_tiles = (int64_t)p.tiles_x * p.tiles_y * p.tiles_t * g.mt * inst;
    LVG_REQUIRE(p.total_tiles < (1ll << 31), "convnd: too many tiles");
    p.div_x = fast_div(p.tiles_x); p.div_y = fast_div(p.tiles_y); p.div_t = fast_div(p.tiles_t); p.div_mt = fast_div(g.mt);
    p.div_groups = fast_div(j.groups);
    // the epilogue places a tile on the stored grid by its tile indices
    LVG_REQUIRE((p.tiles_x == 1 || p.wt % ostride == 0) && (p.tiles_y == 1 || p.th % ostride == 0), "convnd: tile origins off the stride lattice");
    p.ths = p.th / ostride; p.wts = p.wt / ostride;
    p.pair_store = plan_pairs_columns(p) ? 1 : 0;          // run_igemm clears it for a y that is not aligned for pairs
    return LVG_OK;
}

}  // namespace

bool ConvShape::tileable() const { return nd_supported(dtype, kt, kh, kw) && n >= 1 && groups >= 1; }
bool ConvShape::fprop_ok() const { return tileable() && pad_t >= 0 && pad_h >= 0 && pad_w >= 0 && stride >= 1 && stride <= 4; }
bool ConvShape::dgrad_ok() const { return fprop_ok() && pad_t <= kt - 1 && pad_h <= kh - 1 && pad_w <= kw - 1; }
bool ConvShape::wgrad_ok() const { return fprop_ok() && kw <= 3 && !empty() && wo() <= 4 * (128 - kw + 1); }

Geometry geometry(int split, int64_t inst, int groups, int ck, int cm, int64_t thw, int taps)
{
    Geometry g;
    g.cpad = round_up(ck, 16);
    g.cblk = g.cpad / 8;
    g.nblk = split ? 2 * g.cblk : g.cblk;
    g.nimg = split ? 2 : 1;
    g.kc = g.cpad / 16;
    g.mt = (cm + kBM - 1) / kBM;
    // at most 64 rows: 64-row weight images (half the A bytes per stage, no all-zero MMA rows)
    g.m64 = cm <= 64 && env_flag("LVG_CONV_M64", 1) ? 1 : 0;
    g.a_img = g.m64 ? kATile / 2 : kATile;
    g.act_bytes = inst * g.nblk * thw * 16;
    g.w_bytes = (int64_t)groups * g.mt * g.kc * taps * g.nimg * g.a_img;
    return g;
}

IgemmJob fprop_job(const ConvShape& s, const void* x, const void* w, void* y)
{
    IgemmJob j = {};
    j.x = x; j.xin_h = s.h; j.xin_w = s.wd; j.dil = 1;
    j.dtype = s.dtype; j.n = s.n; j.groups = s.groups; j.ck = s.cin; j.cm = s.cout;
    j.t = s.t; j.h = s.h; j.wd = s.wd; j.kt = s.kt; j.kh = s.kh; j.kw = s.kw; j.pad_t = s.pad_t; j.pad_h = s.pad_h; j.pad_w = s.pad_w;
    j.w = w; j.gs = (int64_t)s.cout * s.cin * s.taps(); j.sm = (int64_t)s.cin * s.taps(); j.sk = s.taps(); j.flip = 0;
    j.y = y; j.gain = 1.f; j.clamp = -1.f;
    j.ostride = s.stride;
    return j;
}

// The input gradient as a forward convolution: dy (to x ho x wo, cout channels; for a strided convolution dy is spread
// over every stride-th pixel of that grid) with the channel-transposed, mirrored weights, padding k - 1 - pad.
IgemmJob dgrad_job(const ConvShape& s, const void* dy, const void* w, void* dx)
{
    IgemmJob j = {};
    j.x = dy; j.xin_h = s.hos(); j.xin_w = s.wos(); j.dil = s.stride;
    j.dtype = s.dtype; j.n = s.n; j.groups = s.groups; j.ck = s.cout; j.cm = s.cin;
    j.t = s.to(); j.h = s.ho(); j.wd = s.wo(); j.kt = s.kt; j.kh = s.kh; j.kw = s.kw;
    j.pad_t = s.kt - 1 - s.pad_t; j.pad_h = s.kh - 1 - s.pad_h; j.pad_w = s.kw - 1 - s.pad_w;
    j.w = w; j.gs = (int64_t)s.cout * s.cin * s.taps(); j.sm = s.taps(); j.sk = (int64_t)s.cin * s.taps(); j.flip = 1;
    j.y = dx; j.gain = 1.f; j.clamp = -1.f;
    j.ostride = 1;
    return j;
}

IgemmRooms igemm_rooms(const IgemmJob& j) { return igemm_rooms_of(job_geometry(j), j.x8_pre != nullptr); }

// plan, re-tile the operands (x unless pre-tiled, the weights always) into the workspace, launch
int run_igemm(const IgemmJob& j, void* workspace, int64_t workspace_bytes, cudaStream_t s)
{
    IgemmParams p;
    const int prc = plan_igemm(j, p);
    if (prc) return prc;
    const int split = j.dtype == LVG_F32 ? 1 : 0;
    const int taps = j.kt * j.kh * j.kw;
    const int64_t inst = (int64_t)j.n * j.groups;
    const Geometry g = job_geometry(j);
    const IgemmRooms r = igemm_rooms_of(g, j.x8_pre != nullptr);
    LVG_REQUIRE(workspace && workspace_bytes >= r.total(), "convnd: workspace too small");
    LVG_REQUIRE(aligned16(workspace), "convnd: workspace must be 16-byte aligned");
    LVG_REQUIRE(encode_fn() != nullptr, "convnd: cuTensorMapEncodeTiled is not available from this driver");
    unsigned char* wp = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* x8 = j.x8_pre ? const_cast<unsigned char*>(j.x8_pre) : wp + r.wp;
    p.wp = wp;
    if (reinterpret_cast<uintptr_t>(j.y) % (split ? 8 : 4) != 0) p.pair_store = 0;

    // re-tile the operands
    {
        const int rc = j.x8_pre ? LVG_OK : pack_act(j.x, x8, split, inst, j.ck, g.cblk, j.t, j.xin_h, j.xin_w, j.h, j.wd, j.dil, s, j.in_scale, &j.in_gate);
        if (rc) return rc;
        const int64_t wblocks = (int64_t)j.groups * g.mt * g.kc;
        LVG_REQUIRE(wblocks < (1ll << 31), "convnd: too many weight tiles");
        // rows of m per pass: <= ~64 KB of staging (16 * rows * taps elements either way)
        const int es = split ? 4 : 2;
        const int img_rows = g.m64 ? 64 : kBM;
        int rpp = (int)((64 * 1024) / (16 * taps * es + 16)) / 8 * 8;
        if (rpp > img_rows) rpp = img_rows;
        if (rpp < 8) rpp = 8;
        const bool mrows = j.sk < j.sm;
        const int run_el = mrows ? 16 * taps : rpp * taps;
        const int pitch = ((run_el * es + 2 + 3) / 4) | 1;
        const int max_runs = mrows ? rpp : 16;
        const size_t wsm = ((size_t)max_runs * pitch + max_runs + 4) * 4;
        // row chunks per image: enough CTAs for two per SM (1, 2, 4 or 8 chunks of img_rows / chunks rows)
        int chunks = 1;
        {
            const char* e = getenv("LVG_PACKW_CHUNKS");       // experiments
            if (e && atoi(e) >= 1) chunks = atoi(e) >= 8 ? 8 : (atoi(e) >= 4 ? 4 : (atoi(e) >= 2 ? 2 : 1));
            else while (chunks < 8 && wblocks * chunks < 2 * (int64_t)num_sms()) chunks *= 2;
        }
        const int rows_per_cta = img_rows / chunks;
        const dim3 wgrid((unsigned)wblocks, (unsigned)chunks);
        if (split) {
            LVG_CUDA(cudaFuncSetAttribute(conv_pack_w_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            conv_pack_w_kernel<float, true><<<wgrid, 256, wsm, s>>>((const float*)j.w, wp, j.cm, j.ck, g.cpad, taps, j.gs, j.sm, j.sk, j.flip, g.mt,
                                                                    g.kc, rpp, rows_per_cta, img_rows);
        } else {
            LVG_CUDA(cudaFuncSetAttribute(conv_pack_w_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            conv_pack_w_kernel<__half, false><<<wgrid, 256, wsm, s>>>((const __half*)j.w, wp, j.cm, j.ck, g.cpad, taps, j.gs, j.sm, j.sk, j.flip,
                                                                      g.mt, g.kc, rpp, rows_per_cta, img_rows);
        }
        LVG_LAUNCH_CHECK();
    }

    // tensor map over X8 as 8-byte elements: (2 W, H, T, instance * block)
    CUtensorMap tm;
    {
        const int rc = encode_map(&tm, x8, j.wd, j.h, j.t, inst * g.nblk, j.wd, (int64_t)j.h * j.wd, (int64_t)j.t * j.h * j.wd, p.wtb, p.thb,
                                  p.tt, 2);
        if (rc) return rc;
    }
    const size_t smem = (size_t)igemm_smem_bytes(p);
    // one instantiation per MMA width (the output-scaled epilogue is a separate one: the unscaled one stays as it was)
#define LVG_IGEMM_WIDTHS(B, S)                                                                                                     \
    {conv_igemm_kernel<B, 16, S>,  conv_igemm_kernel<B, 32, S>,  conv_igemm_kernel<B, 48, S>,  conv_igemm_kernel<B, 64, S>,        \
     conv_igemm_kernel<B, 80, S>,  conv_igemm_kernel<B, 96, S>,  conv_igemm_kernel<B, 112, S>, conv_igemm_kernel<B, 128, S>,       \
     conv_igemm_kernel<B, 144, S>, conv_igemm_kernel<B, 160, S>, conv_igemm_kernel<B, 176, S>, conv_igemm_kernel<B, 192, S>,       \
     conv_igemm_kernel<B, 208, S>, conv_igemm_kernel<B, 224, S>, conv_igemm_kernel<B, 240, S>, conv_igemm_kernel<B, 256, S>}
    void (*const kerns[2][2][kWidths])(const CUtensorMap, const IgemmParams) = {
        {LVG_IGEMM_WIDTHS(false, false), LVG_IGEMM_WIDTHS(true, false)}, {LVG_IGEMM_WIDTHS(false, true), LVG_IGEMM_WIDTHS(true, true)}};
#undef LVG_IGEMM_WIDTHS
    LVG_REQUIRE(p.ncw % 16 == 0 && p.ncw >= 16 && p.ncw <= 16 * kWidths, "convnd: MMA width %d", p.ncw);
    void (*kern)(const CUtensorMap, const IgemmParams) = kerns[j.out_scale != nullptr][split][p.ncw / 16 - 1];
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const char* cta_env = getenv("LVG_CONV_CTAS");          // experiments: fewer persistent CTAs than SMs
    const int max_ctas = cta_env ? atoi(cta_env) : num_sms();
    int64_t ctas = p.total_tiles < max_ctas ? p.total_tiles : max_ctas;
    kern<<<(unsigned)ctas, kIgemmThreads, smem, s>>>(tm, p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_convnd_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                        int pad_t, int pad_h, int pad_w)
{
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!sh.tileable() || sh.empty()) return -1;
    // the engine's forward and input gradient, and the pointwise wgmma kernels (which pack their weights here) in both roles
    return std::max(std::max(igemm_rooms(fprop_job(sh, nullptr, nullptr, nullptr)).total(), igemm_rooms(dgrad_job(sh, nullptr, nullptr, nullptr)).total()),
                    std::max(pw_tc_workspace(dtype, cin, cout), pw_tc_workspace(dtype, cout, cin)));
}

extern "C" int lvg_convnd_fprop(const void* x, const void* w, void* y, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                                int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, const float* bias, int act, float alpha,
                                float gain, float clamp, void* workspace, int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && w && y, "convnd_fprop: x, w, y must not be NULL");
    const int route = lvg_convnd_route(0, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride,
                                       bias || act != 0 || gain != 1.f || clamp >= 0.f);
    if (route == 1) return pw_conv((const float*)x, (const float*)w, (float*)y, n, cin, cout, (int64_t)t * h * wd, cin, 1, (cudaStream_t)stream);
    if (route == 2 && aligned16(x) && aligned16(y))
        return pw_tc_conv(x, w, y, dtype, n, cin, cout, (int64_t)t * h * wd, cin, 1, workspace, workspace_bytes, (cudaStream_t)stream);
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    if (!sh.fprop_ok()) {
        set_error("convnd_fprop: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    IgemmJob j = fprop_job(sh, x, w, y);
    j.bias = bias; j.act = act; j.alpha = alpha; j.gain = gain; j.clamp = clamp;
    return run_igemm(j, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int lvg_convnd_dgrad(const void* dy, const void* w, void* dx, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                                int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, void* workspace, int64_t workspace_bytes,
                                void* stream)
{
    LVG_REQUIRE(dy && w && dx, "convnd_dgrad: dy, w, dx must not be NULL");
    const int route = lvg_convnd_route(1, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, 0);     // dx = W^T dy
    if (route == 1) return pw_conv((const float*)dy, (const float*)w, (float*)dx, n, cout, cin, (int64_t)t * h * wd, 1, cin, (cudaStream_t)stream);
    if (route == 2 && aligned16(dy) && aligned16(dx))
        return pw_tc_conv(dy, w, dx, dtype, n, cout, cin, (int64_t)t * h * wd, 1, cin, workspace, workspace_bytes, (cudaStream_t)stream);
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    if (!sh.dgrad_ok()) {
        set_error("convnd_dgrad: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    return run_igemm(dgrad_job(sh, dy, w, dx), workspace, workspace_bytes, (cudaStream_t)stream);
}


// =================================================================================================
// Weight gradient:  dW[g][co][ci][kt][ky][kx] = sum over samples and output pixels of dy[co][pix] * x[ci][pix + tap]
//
// GEMM view per CTA (group g, 128-channel tile of co, NT-channel tile of ci, tap row (kt, ky)):
//   D_kx[co][ci] += A[co][k] * B_kx[ci][k],   K = output pixels, the kw taps of the row as kw register accumulators.
// Both operands come from the SAME channel-block-of-8 tensors the forward kernels use, now as MN-major operands: a pixel
// is a 16-byte row (8 channels) and the pixel index runs linearly at 16 bytes over a stage tile of RH rows x PS columns,
// PS = (segment width + kw - 1) rounded up to 16. The dy tile is loaded through a tensor map whose W extent is clipped to
// the column segment, so TMA zero-fills its last PS - width columns -- those are the K positions where the x tile holds
// the row's halo; with equal pitches on both sides a tap (kx) is a start-address shift of kx * 16 bytes and the tap row
// (kt, ky) a shifted TMA box. One MMA covers 16 consecutive pixels of the linear index.
// Few groups (discriminators, low-res networks): the stages are cut into `nsplit` ranges over the grid, fp32 partial
// sums go to a workspace and conv_wgrad_reduce_kernel folds them. fp32 tensors: hi/lo bf16 halves of BOTH operands are
// staged, three MMAs per k-step (hi*hi + lo*hi + hi*lo).

namespace lvg {
namespace {

struct WgradV2Params {
    void* dw;                    // final output when nsplit == 1, else fp32 partials [nsplit][...]
    int out_f32;                 // element type of `dw` (partials are always fp32)
    int bf16, split;             // operand format; split = hi/lo pairs staged
    int n, groups, cin, cout;
    int to, ho;                  // output rows / frames iterated
    int kt, kh, kw, pad_t, pad_h, pad_w;
    int nt;                      // ci per n-tile (multiple of 16)
    int nblk_a, nblk_b;          // channel blocks per instance in dy8 / x8 (incl. the lo half in split mode)
    int lo_a, lo_b;              // block offset of the lo half
    int nseg, seg_w[4], seg_x0[4], ps[4];
    int rh;                      // dy rows per stage
    int khc;                     // tap rows (ky) per CTA: 1, or kh (folded: one dy tile and one x tile of rh + kh - 1 rows serve all ky)
    int ablk;                    // channel blocks of one dy image in a stage (16, or fewer for cout < 128: the rest of the 128 MMA rows is never stored)
    int nsplit;
    int a_bytes, b_bytes, stage_bytes, stages;      // per stage: one A (B) operand image; a stage holds split+1 of each
    int64_t split_stride;        // elements between fp32 partials
    int mrows;                   // output-channel rows computed: 128, or 64 (cout <= 64: one consumer warpgroup)
    int tail_bytes;              // shared memory behind the stage ring that the MMAs may read (kx-shifted last rows; the 128 - 8 * ablk rows without data)
};

struct WgradMaps { CUtensorMap a[4]; CUtensorMap b; };     // dy8 clipped to each column segment; x8

// Roles (384 threads): warp 0 = TMA producer (one lane); warpgroups 1 and 2 = MMA + epilogue for output channels 0-63 and
// 64-127 of the m-tile (only the first when mrows = 64). A consumer holds the TAPS = khc * kw accumulators of NT columns
// each in registers (TAPS * NT <= 256) and issues one m64nNTk16 per tap and k step: the x-tile descriptor steps over the
// NT / 8 channel blocks with its stride byte offset.
template <bool BF16, int TAPS, int NT>
__global__ void __launch_bounds__(kIgemmThreads, 1) conv_wgrad_v2_kernel(const __grid_constant__ WgradMaps maps, const WgradV2Params p)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);

    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);
    int bx = blockIdx.x;
    const int sp = bx % p.nsplit; bx /= p.nsplit;
    int ky0 = 0;
    if (p.khc == 1) { ky0 = bx % p.kh; bx /= p.kh; }
    const int kt = bx % p.kt;
    const int nti = bx / p.kt;
    const int mti = blockIdx.y, g = blockIdx.z;
    const int nop = p.split ? 2 : 1;                              // operand images per stage and side
    const int consumers = p.mrows / 64;

    // stages of this CTA: (sample, frame, segment, row block), range [s0, s1)
    const int rblocks = (p.ho + p.rh - 1) / p.rh;
    const int per_plane = p.nseg * rblocks;
    const int total = p.n * p.to * per_plane;
    const int s0 = (int)((int64_t)total * sp / p.nsplit), s1 = (int)((int64_t)total * (sp + 1) / p.nsplit);

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], (uint32_t)consumers); }
        fence_barrier_init();
    }
    // zero the slack behind the stage buffers (the kx-shifted reads of the last block run 32 bytes past its end; the dy
    // values they meet are zero, and zero * garbage must not become NaN)
    // (uninitialised shared memory may hold NaN patterns: clear all of it once)
    for (int i = threadIdx.x; i < (p.stages * p.stage_bytes + p.tail_bytes) / 16; i += kIgemmThreads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async();
    __syncthreads();

    if (wg == 0) {
        if (warp == 0 && elect_one()) {
            for (int s = s0; s < s1; s++) {
                const int it = s - s0, slot = it % p.stages;
                if (it >= p.stages) mbar_wait(&empty_bar[slot], (uint32_t)((it / p.stages - 1) & 1));
                int r = s;
                const int rb = r % rblocks; r /= rblocks;
                const int seg = r % p.nseg; r /= p.nseg;
                const int t = r % p.to;
                const int n = r / p.to;
                const int inst = n * p.groups + g;
                unsigned char* st = smem + (size_t)slot * p.stage_bytes;
                mbar_expect_tx(&full_bar[slot], (uint32_t)(nop * (p.a_bytes + p.b_bytes)));
                const int oy0 = rb * p.rh;
                for (int o = 0; o < nop; o++) {
                    tma_load_4d(st + (size_t)o * p.a_bytes, &maps.a[seg], 0, oy0, t, inst * p.nblk_a + o * p.lo_a + mti * 16, &full_bar[slot]);
                    tma_load_4d(st + (size_t)nop * p.a_bytes + (size_t)o * p.b_bytes, &maps.b, 2 * (p.seg_x0[seg] - p.pad_w), oy0 + ky0 - p.pad_h,
                                t + kt - p.pad_t, inst * p.nblk_b + o * p.lo_b + nti * (NT / 8), &full_bar[slot]);
                }
            }
        }
    } else if (wg >= 1 && wg - 1 < consumers) {
        const int cw = wg - 1;
        const int tid = threadIdx.x % 128, wq = tid / 32;
        float acc[TAPS][NT / 2];
#pragma unroll
        for (int tap = 0; tap < TAPS; tap++)
#pragma unroll
            for (int i = 0; i < NT / 2; i++) acc[tap][i] = 0.f;
        int prev = -1;
        for (int s = s0; s < s1; s++) {
            const int it = s - s0, slot = it % p.stages;
            const int seg = (s / rblocks) % p.nseg;
            const int rb = s % rblocks;
            const int rows = min(p.rh, p.ho - rb * p.rh);
            const int ksteps = (rows * p.ps[seg] + 15) / 16;                 // (a trailing half step reads the zero-filled next row)
            const uint32_t blk_a = (uint32_t)(p.rh * p.ps[seg] * 16);                    // bytes of one channel block of the dy tile
            const uint32_t blk_b = (uint32_t)((p.rh + p.khc - 1) * p.ps[seg] * 16);      // ... of the x tile (kh - 1 halo rows when folded)
            const uint32_t ky16 = (uint32_t)p.ps[seg];                                   // one tap row down = one tile row further (>> 4)
            mbar_wait(&full_bar[slot], (uint32_t)((it / p.stages) & 1));
            wgmma_fence();
            const uint32_t a0 = smem_u32(smem + (size_t)slot * p.stage_bytes) + (uint32_t)cw * 8u * blk_a;
            const uint32_t b0 = smem_u32(smem + (size_t)slot * p.stage_bytes) + (uint32_t)(nop * p.a_bytes);
            // descriptors as (lo, hi) words: a K step is +16 on the low word (256 bytes >> 4), a tap column +1, a tap row
            // + ps; the stride byte offset of the x tile (one channel block) spans the NT / 8 blocks of the n-tile
            const uint32_t a_hi = desc_hi(blk_a), b_hi = desc_hi(blk_b);
            for (int term = 0; term < (p.split ? 3 : 1); term++) {
                const uint32_t a_lo0 = desc_lo(a0 + (term == 1 ? (uint32_t)p.a_bytes : 0u), 128);     // hi*hi, lo*hi, hi*lo
                const uint32_t b_lo0 = desc_lo(b0 + (term == 2 ? (uint32_t)p.b_bytes : 0u), 128);
                for (int k = 0; k < ksteps; k++) {
#pragma unroll
                    for (int tap = 0; tap < TAPS; tap++) {
                        const int kyi = tap / p.kw, kx = tap - kyi * p.kw;
                        wgmma_m64nNk16<BF16, NT, 1, 1>(acc[tap], a_lo0 + 16u * k, a_hi, b_lo0 + 16u * k + (uint32_t)kyi * ky16 + (uint32_t)kx, b_hi);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                              // the group of the previous stage has completed: release its slot
            mbar_arrive_if(&empty_bar[prev >= 0 ? prev : 0], prev >= 0 && tid == 0);
            prev = slot;
        }
        wgmma_wait<0>();

        // ---- epilogue: registers -> dW[g][co][ci][kt][ky][kx] (or the fp32 partial sums of split `sp`)
        const int taps = p.kt * p.kh * p.kw;
        const int ci0 = nti * NT;
#pragma unroll
        for (int tap = 0; tap < TAPS; tap++) {
            const int kyi = tap / p.kw, kx = tap - kyi * p.kw;
            const int tapg = (kt * p.kh + ky0 + kyi) * p.kw + kx;
#pragma unroll
            for (int i = 0; i < NT / 2; i++) {
                const int co = mti * kBM + cw * 64 + wq * 16 + lane / 4 + 8 * ((i / 2) % 2);
                const int cil = (i / 4) * 8 + 2 * (lane % 4) + i % 2;
                if (co >= p.cout || ci0 + cil >= p.cin) continue;
                const int64_t off = (((int64_t)g * p.cout + co) * p.cin + ci0 + cil) * taps + tapg;
                const float v = acc[tap][i];
                if (p.nsplit > 1) reinterpret_cast<float*>(p.dw)[(int64_t)sp * p.split_stride + off] = v;
                else if (p.out_f32) reinterpret_cast<float*>(p.dw)[off] = v;
                else reinterpret_cast<__half*>(p.dw)[off] = __float2half_rn(v);
            }
        }
    }
}

template <class TOut>
__global__ void __launch_bounds__(256) conv_wgrad_reduce_kernel(const float* __restrict__ part, TOut* __restrict__ out, int64_t n, int nsplit, int64_t stride)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < nsplit; k++) s += part[(int64_t)k * stride + i];
        if constexpr (sizeof(TOut) == 2) out[i] = __float2half_rn(s);
        else out[i] = s;
    }
}

// channel padding of the dy8 operand of the weight gradient. cout < 128: only the channel blocks that exist (the same
// tensor the input gradient reads, so one re-tiling pass serves both; the remaining rows of the 128-row MMA read whatever
// follows in shared memory and are never stored -- rows of D depend on the same rows of A only). Otherwise whole m-tiles.
inline int wgrad_cpad_a(int cout) { return (cout < kBM && env_flag("LVG_WGRAD_COMPACT", 1)) ? round_up(cout, 16) : round_up(cout, kBM); }

}  // namespace

WgradPlan wgrad_plan(const ConvShape& s, bool fold)
{
    const int cin = s.cin, cout = s.cout, kh = s.kh, kw = s.kw;
    const int to = s.to(), ho = s.ho(), wo = s.wo();
    WgradPlan q;
    q.split = s.split();
    q.cpad_a = wgrad_cpad_a(cout);
    q.ablk = q.cpad_a < kBM ? q.cpad_a / 8 : 16;
    // rows of the accumulator: with at most 64 output channels one consumer warpgroup (M = 64) does all the work
    q.mrows = (q.cpad_a <= 64 && env_flag("LVG_WGRAD_M64", 1)) ? 64 : kBM;
    q.cpad_b = round_up(cin, 16);
    // Few input channels (<= 32): ONE CTA takes all kh tap rows -- the x tile carries kh - 1 halo rows and a tap row is a
    // start-address shift of one tile row, like kx is a shift of one pixel -- so dy and x are fetched once per (kt, n-tile)
    // instead of once per (kt, ky), where the kh * kw accumulators of 32 columns each fit the 256 register columns of a
    // consumer warpgroup (kh * kw <= 8).
    q.khc = (fold && kh > 1 && kh * kw * 32 <= 256 && cin <= env_flag("LVG_WGRAD_FOLD_CIN", 32) && env_flag("LVG_WGRAD_FOLD", 1)) ? kh : 1;
    int nt_cap = (256 / (q.khc * kw)) / 32 * 32;
    if (q.split && nt_cap > 128) nt_cap = 128;
    // column segments (a TMA box row is at most 128 pixels incl. the kw - 1 halo) and the common tile pitch
    q.nseg = (wo + 128 - kw) / (129 - kw);
    if (q.nseg < 1) q.nseg = 1;
    const int w0 = (wo + q.nseg - 1) / q.nseg;
    for (int j = 0; j < 4; j++) { q.seg_x0[j] = j * w0; q.seg_w[j] = j < q.nseg ? (wo - j * w0 < w0 ? wo - j * w0 : w0) : 0; }
    q.ps = round_up(w0 + kw - 1, 8);                           // rows x pitch must be a multiple of 16 pixels (one MMA K step)
    const int nop = q.split ? 2 : 1;
    // bytes of a stage with `rows` dy rows and an n-tile of `nt` channels
    auto stage_of = [&](int rows, int nt) { return nop * (q.ablk * rows + (nt / 8) * (rows + q.khc - 1)) * q.ps * 16; };
    {   // a pitch of 8 mod 16 needs row pairs: take it only when two stages of two rows fit with a useful n-tile
        if (q.ps % 16 != 0 && 2 * stage_of(2, 64 < nt_cap ? 64 : nt_cap) > 200 * 1024) q.ps = round_up(q.ps, 16);
    }
    {   // the smallest stage (1 or 2 rows) must leave room for two stages
        const int min_rows = q.ps % 16 != 0 ? 2 : 1;
        while (nt_cap > 32 && 2 * stage_of(min_rows, nt_cap) > 200 * 1024) nt_cap -= 32;
    }
    q.ntiles = (q.cpad_b + nt_cap - 1) / nt_cap;
    q.nt = round_up((q.cpad_b + q.ntiles - 1) / q.ntiles, 32);          // the MMAs take the input channels 32 at a time
    q.cpad_b = q.nt * q.ntiles;
    q.mt = (q.cpad_a + kBM - 1) / kBM;
    const int64_t inst = s.inst();
    q.a_bytes = inst * nop * (q.cpad_a / 8) * (int64_t)to * ho * wo * 16;
    q.b_bytes = inst * nop * (q.cpad_b / 8) * s.thw() * 16;
    q.dw_elems = (int64_t)s.groups * cout * cin * s.taps();
    // rows per stage: about 80 KB of operands per stage
    q.rh = 1;
    while (q.rh < ho && q.rh < 255 - q.khc && stage_of(q.rh + 1, q.nt) <= 80 * 1024) q.rh++;
    if (q.ps % 16 != 0) q.rh = q.rh >= 2 ? q.rh / 2 * 2 : 2;   // even row count (rows past the image are zero-filled)
    // behind the ring: the kx-shifted reads of the last block (32 bytes) and, with fewer dy blocks than the MMA has rows / 8,
    // the rows beyond them (read from the lo image's start: (nop - 1) * a_stage + mrows / 8 blocks). Two stages + tail must fit.
    for (;;) {
        q.a_stage = q.ablk * q.rh * q.ps * 16;
        q.b_stage = (q.nt / 8) * (q.rh + q.khc - 1) * q.ps * 16;
        q.stage_bytes = round_up(nop * (q.a_stage + q.b_stage), 128);
        const int over = (nop - 1) * q.a_stage + (q.mrows / 8) * q.rh * q.ps * 16 - q.stage_bytes;
        q.tail_bytes = round_up(256 + (over > 0 ? over : 0), 128);
        const int step = q.ps % 16 != 0 ? 2 : 1;
        if (2 * q.stage_bytes + q.tail_bytes <= 220 * 1024 || q.rh <= step) break;
        q.rh -= step;
    }
    q.stages = 2;
    while (q.stages < kMaxStages && (q.stages + 1) * q.stage_bytes + q.tail_bytes <= 220 * 1024) q.stages++;
    q.smem = (size_t)q.stages * q.stage_bytes + q.tail_bytes + 128;
    // tall folded kernels (7 or 8 tap rows) over wide rows in split precision: even one-row stages of NT = 32 overflow shared
    // memory with the x tile's kh - 1 halo rows -- one CTA per tap row instead
    if (q.khc > 1 && q.smem > 227 * 1024) return wgrad_plan(s, false);
    // Split the pixel range over `nsplit` CTAs per output tile. One CTA per SM is resident, so the kernel runs in waves of
    // num_sms CTAs: choose the split that minimises waves x (stages per CTA + a fixed per-CTA cost of ~4 stages: clearing
    // shared memory, the register -> global epilogue) -- e.g. with 132 SMs and 3 output tiles: 44 splits = 132 CTAs = one
    // wave instead of 64 splits = 192 CTAs = two waves. Partial sums are capped at 256 MB.
    const int64_t ctas = (int64_t)q.ntiles * (kh / q.khc) * s.kt * q.mt * s.groups;
    const int64_t stages = (int64_t)s.n * to * q.nseg * ((ho + q.rh - 1) / q.rh);
    const int sms = num_sms();
    int64_t cap = 160;
    if (cap > stages) cap = stages;
    while (cap > 1 && cap * q.dw_elems * 4 > (256ll << 20)) cap--;
    int64_t ns = 1;
    double best = 1e300;
    for (int64_t k = 1; k <= cap; k++) {
        const int64_t waves = (ctas * k + sms - 1) / sms;
        const double tm = (double)waves * ((double)((stages + k - 1) / k) + 4.0 * q.khc);
        if (tm < best * 0.999) { best = tm; ns = k; }
    }
    {
        const char* e = getenv("LVG_WGRAD_NSPLIT");       // experiments
        if (e && atoi(e) >= 1) ns = atoi(e) < stages ? atoi(e) : stages;
    }
    q.nsplit = (int)ns;
    q.part_bytes = q.nsplit > 1 ? q.nsplit * q.dw_elems * 4 : 0;
    return q;
}

namespace {

// The (taps per CTA, NT) pairs wgrad_plan can return: NT a multiple of 32 with taps * NT <= 256 (kw <= 3, and kh * kw <= 8
// when the tap rows are folded), NT <= 128 with split operands. nullptr for anything else.
typedef void (*WgradKernel)(const WgradMaps, const WgradV2Params);
template <bool B>
WgradKernel wgrad_kernel_of(int taps, int nt)
{
    switch (taps * 1000 + nt) {
    case 1032: return conv_wgrad_v2_kernel<B, 1, 32>;
    case 1064: return conv_wgrad_v2_kernel<B, 1, 64>;
    case 1096: return conv_wgrad_v2_kernel<B, 1, 96>;
    case 1128: return conv_wgrad_v2_kernel<B, 1, 128>;
    case 2032: return conv_wgrad_v2_kernel<B, 2, 32>;
    case 2064: return conv_wgrad_v2_kernel<B, 2, 64>;
    case 2096: return conv_wgrad_v2_kernel<B, 2, 96>;
    case 2128: return conv_wgrad_v2_kernel<B, 2, 128>;
    case 3032: return conv_wgrad_v2_kernel<B, 3, 32>;
    case 3064: return conv_wgrad_v2_kernel<B, 3, 64>;
    case 4032: return conv_wgrad_v2_kernel<B, 4, 32>;
    case 4064: return conv_wgrad_v2_kernel<B, 4, 64>;
    case 5032: return conv_wgrad_v2_kernel<B, 5, 32>;
    case 6032: return conv_wgrad_v2_kernel<B, 6, 32>;
    case 7032: return conv_wgrad_v2_kernel<B, 7, 32>;
    case 8032: return conv_wgrad_v2_kernel<B, 8, 32>;
    }
    if constexpr (!B) {
        switch (taps * 1000 + nt) {
        case 1160: return conv_wgrad_v2_kernel<B, 1, 160>;
        case 1192: return conv_wgrad_v2_kernel<B, 1, 192>;
        case 1224: return conv_wgrad_v2_kernel<B, 1, 224>;
        case 1256: return conv_wgrad_v2_kernel<B, 1, 256>;
        }
    }
    return nullptr;
}
WgradKernel wgrad_kernel(int split, int taps, int nt) { return split ? wgrad_kernel_of<true>(taps, nt) : wgrad_kernel_of<false>(taps, nt); }

// the tiles of dy and x agree (cout < 128 or a multiple of 128: every layer of the networks), so one re-tiling of dy can
// serve the input gradient and the weight gradient
bool dy8_tiles_agree(const ConvShape& s) { return wgrad_cpad_a(s.cout) == round_up(s.cout, 16); }

}  // namespace

WgradRooms wgrad_rooms(const WgradPlan& q, bool dy8_pre) { return {dy8_pre ? 0 : round256(q.a_bytes), round256(q.b_bytes), q.part_bytes}; }

int run_wgrad(const ConvShape& sh, const void* x, const void* dy, void* dw, const WgradInputs& in, void* workspace, int64_t workspace_bytes,
              cudaStream_t s)
{
    const int to = sh.to(), ho = sh.ho(), wo = sh.wo();
    const WgradPlan q = wgrad_plan(sh);
    const WgradRooms r = wgrad_rooms(q, in.dy8_pre != nullptr);
    LVG_REQUIRE(workspace && workspace_bytes >= r.total(), "convnd_wgrad: workspace too small");
    LVG_REQUIRE(aligned16(workspace), "convnd_wgrad: workspace must be 16-byte aligned");
    LVG_REQUIRE(sh.groups <= 65535 && q.mt <= 65535, "convnd_wgrad: too many groups / channel tiles");
    const int64_t inst = sh.inst();
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* dy8 = in.dy8_pre ? const_cast<unsigned char*>(in.dy8_pre) : ws;
    unsigned char* x8 = in.x8_pre ? const_cast<unsigned char*>(in.x8_pre) : ws + r.dy8;
    float* part = reinterpret_cast<float*>(ws + r.dy8 + r.x8);
    const int64_t thw_a = (int64_t)to * ho * wo, thw_b = sh.thw();
    {
        // dy of a strided convolution is spread over every stride-th pixel of the stride-1 output grid (zeros between)
        int rc = in.dy8_pre ? LVG_OK : pack_act(dy, dy8, q.split, inst, sh.cout, q.cpad_a / 8, to, sh.hos(), sh.wos(), ho, wo, sh.stride, s, in.dy_scale,
                                                &in.dy_gate);
        if (rc) return rc;
        rc = in.x8_pre ? LVG_OK : pack_act(x, x8, q.split, inst, sh.cin, q.cpad_b / 8, sh.t, sh.h, sh.wd, sh.h, sh.wd, 1, s, in.x_scale);
        if (rc) return rc;
    }
    WgradV2Params p;
    memset(&p, 0, sizeof(p));
    p.out_f32 = q.split; p.bf16 = q.split; p.split = q.split;
    p.n = sh.n; p.groups = sh.groups; p.cin = sh.cin; p.cout = sh.cout; p.to = to; p.ho = ho;
    p.kt = sh.kt; p.kh = sh.kh; p.kw = sh.kw; p.pad_t = sh.pad_t; p.pad_h = sh.pad_h; p.pad_w = sh.pad_w;
    p.nt = q.nt;
    p.nblk_a = (q.split ? 2 : 1) * (q.cpad_a / 8); p.nblk_b = (q.split ? 2 : 1) * (q.cpad_b / 8);
    p.lo_a = q.cpad_a / 8; p.lo_b = q.cpad_b / 8;
    p.nseg = q.nseg;
    for (int j = 0; j < 4; j++) { p.seg_w[j] = q.seg_w[j]; p.seg_x0[j] = q.seg_x0[j]; p.ps[j] = q.ps; }
    p.rh = q.rh; p.khc = q.khc; p.ablk = q.ablk;
    p.mrows = q.mrows;
    p.a_bytes = q.a_stage; p.b_bytes = q.b_stage; p.stage_bytes = q.stage_bytes; p.stages = q.stages; p.tail_bytes = q.tail_bytes;
    const size_t smem = q.smem;
    LVG_REQUIRE(smem <= 227 * 1024, "convnd_wgrad: stage does not fit shared memory (%zu bytes)", smem);
    p.nsplit = q.nsplit;
    p.split_stride = q.dw_elems;
    p.dw = q.nsplit > 1 ? (void*)part : dw;
    // NOTE the per-segment tile pitch: a stage tile of segment j is [block][rows][ps[j]][16 B] -- the box width IS the pitch
    WgradMaps maps;
    memset(&maps, 0, sizeof(maps));
    for (int j = 0; j < p.nseg; j++) {
        const int rc = encode_map(&maps.a[j], dy8 + (size_t)p.seg_x0[j] * 16, p.seg_w[j], ho, to, inst * p.nblk_a, wo, (int64_t)ho * wo, thw_a,
                                  p.ps[j], p.rh, 1, q.ablk);
        if (rc) return rc;
    }
    {
        const int rc = encode_map(&maps.b, x8, sh.wd, sh.h, sh.t, inst * p.nblk_b, sh.wd, (int64_t)sh.h * sh.wd, thw_b, p.ps[0], p.rh + q.khc - 1, 1,
                                  q.nt / 8);
        if (rc) return rc;
    }
    void (*const kern)(const WgradMaps, const WgradV2Params) = wgrad_kernel(q.split, q.khc * sh.kw, q.nt);
    LVG_REQUIRE(kern != nullptr, "convnd_wgrad: no kernel for %d taps x %d columns (split %d)", q.khc * sh.kw, q.nt, q.split);
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((unsigned)(q.ntiles * sh.kt * (sh.kh / q.khc) * q.nsplit), (unsigned)q.mt, (unsigned)sh.groups);
    kern<<<grid, kIgemmThreads, smem, s>>>(maps, p);
    LVG_LAUNCH_CHECK();
    if (q.nsplit > 1) {
        int64_t blocks = (q.dw_elems + 255) / 256;
        const int64_t cap = (int64_t)num_sms() * 32;
        if (blocks > cap) blocks = cap;
        if (q.split) conv_wgrad_reduce_kernel<float><<<(unsigned)blocks, 256, 0, s>>>(part, (float*)dw, q.dw_elems, q.nsplit, q.dw_elems);
        else conv_wgrad_reduce_kernel<__half><<<(unsigned)blocks, 256, 0, s>>>(part, (__half*)dw, q.dw_elems, q.nsplit, q.dw_elems);
        LVG_LAUNCH_CHECK();
    }
    return LVG_OK;
}

// ---- both gradients of one call. dy (times a factor d, for modulated convolutions) is re-tiled ONCE when the tiles of the
// two gradients agree: the input gradient (forward kernel on dy) and the weight gradient (dy as the M-side operand) read
// the same channel-block tensor. LVG_CONV_SHARED_DY8=0 re-tiles it for each gradient.
bool shares_dy8(const ConvShape& s) { return env_flag("LVG_CONV_SHARED_DY8", 1) && dy8_tiles_agree(s); }

BackwardRooms backward_rooms(const ConvShape& s, bool shared)
{
    const Geometry gd = job_geometry(dgrad_job(s, nullptr, nullptr, nullptr));
    const WgradRooms wr = wgrad_rooms(wgrad_plan(s), shared);
    return {shared ? round256(gd.act_bytes) : 0, std::max(igemm_rooms_of(gd, shared).total(), wr.total()), wr.dy8};
}

int64_t backward_workspace(const ConvShape& s)
{
    const int64_t sep = backward_rooms(s, false).total();
    return dy8_tiles_agree(s) ? std::max(sep, backward_rooms(s, true).total()) : sep;
}

int backward_dgrad(const ConvShape& s, const void* dy, const float* d, const void* w, void* dx, void* workspace, int64_t workspace_bytes,
                   cudaStream_t st, Backward& b, const ActGate* gate)
{
    const bool shared = shares_dy8(s);
    const BackwardRooms r = backward_rooms(s, shared);
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.total(), "convnd backward: workspace too small or misaligned");
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    b.dy8 = shared ? ws : nullptr;
    b.rest = ws + r.dy8;
    b.rest_bytes = workspace_bytes - r.dy8;
    b.x8 = b.rest + r.x8;
    b.gate = gate ? *gate : ActGate{};
    IgemmJob j = dgrad_job(s, dy, w, dx);
    if (shared) {
        const int rc = pack_act(dy, ws, s.split(), s.inst(), s.cout, job_geometry(j).cblk, s.to(), s.hos(), s.wos(), s.ho(), s.wo(), s.stride, st, d,
                                &b.gate);
        if (rc) return rc;
        j.x8_pre = ws;
    } else {
        j.in_scale = d;
        j.in_gate = b.gate;
    }
    // (stream order: the weight gradient's re-tiling of x overwrites the packed weights only after the input gradient read them)
    return run_igemm(j, b.rest, b.rest_bytes, st);
}

int backward_wgrad(const ConvShape& s, const Backward& b, const void* x, const void* dy, const float* d, void* dw, const float* x_scale,
                   const unsigned char* x8_pre, cudaStream_t st)
{
    const WgradInputs in = {b.dy8, x8_pre, x_scale, b.dy8 ? nullptr : d, b.dy8 ? ActGate{} : b.gate};
    return run_wgrad(s, x, dy, dw, in, b.rest, b.rest_bytes, st);
}

}  // namespace lvg

extern "C" int64_t lvg_convnd_wgrad_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                              int pad_t, int pad_h, int pad_w)
{
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!sh.wgrad_ok()) return -1;
    return wgrad_rooms(wgrad_plan(sh), false).total();
}

extern "C" int lvg_convnd_wgrad(const void* x, const void* dy, void* dw, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                                int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, void* workspace, int64_t workspace_bytes,
                                void* stream)
{
    LVG_REQUIRE(x && dy && dw, "convnd_wgrad: x, dy, dw must not be NULL");
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    if (!sh.wgrad_ok()) {
        set_error("convnd_wgrad: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    return run_wgrad(sh, x, dy, dw, WgradInputs{}, workspace, workspace_bytes, (cudaStream_t)stream);
}

// which kernels a call takes (host arithmetic only): mode 0 forward (`epilogue` != 0: with a bias / activation / gain /
// clamp epilogue), 1 input gradient, 2 weight gradient -> 0 the engine, 1 the streaming SIMT kernels (conv_pointwise.cu),
// 2 the pointwise wgmma kernels (conv_pw_tc.cu); LVG_UNSUPPORTED outside the envelope. Tensors are taken to be 16-byte
// aligned (the pointwise wgmma route falls back to the engine for a misaligned one).
extern "C" int lvg_convnd_route(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                                int pad_h, int pad_w, int stride, int epilogue)
{
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    if (mode < 0 || mode > 2 || n < 1 || groups < 1) return LVG_UNSUPPORTED;
    if (mode == 2) return sh.wgrad_ok() ? 0 : LVG_UNSUPPORTED;
    if (mode == 1 || !epilogue) {
        if (pw_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, sh.thw())) return 1;
        if (pw_tc_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, sh.thw())) return 2;
    }
    return (mode == 0 ? sh.fprop_ok() : sh.dgrad_ok()) ? 0 : LVG_UNSUPPORTED;
}

// the tiling lvg_convnd_fprop (mode 0) / lvg_convnd_dgrad (mode 1) would launch with, as ints (host arithmetic only;
// tests/test_igemm_emul.py replays the forward kernel's addressing with it on the CPU)
extern "C" int lvg_convnd_plan(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                               int pad_h, int pad_w, int stride, int* out, int out_len)
{
    LVG_REQUIRE(out && out_len >= 48, "convnd_plan: out must hold 48 ints");
    LVG_REQUIRE(mode == 0 || mode == 1, "convnd_plan: mode 0 (forward) or 1 (input gradient)");
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    if (!(mode == 0 ? sh.fprop_ok() : sh.dgrad_ok())) {
        set_error("convnd_plan: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    for (int i = 0; i < out_len; i++) out[i] = 0;
    if (pw_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, sh.thw())) { out[47] = 1; return LVG_OK; }
    if (mode == 1 && sh.empty()) { set_error("convnd_plan: empty output"); return LVG_UNSUPPORTED; }
    IgemmParams p;
    const int rc = plan_igemm(mode == 0 ? fprop_job(sh, nullptr, nullptr, nullptr) : dgrad_job(sh, nullptr, nullptr, nullptr), p);
    if (rc) return rc;
    const int v[48] = {p.wgroups, p.cout, p.mt, p.kc, p.nblk, p.nimg, p.lo_blk, p.to, p.ho, p.wo, p.kt, p.kh, p.kw, p.pad_t, p.pad_h, p.pad_w,
                       p.tt, p.th, p.wt, p.wtb, p.thb, p.frame_px, p.ncols, p.tiles_x, p.tiles_y, p.tiles_t,
                       (int)p.total_tiles, p.ks, p.stages, p.a_resident, p.a_stage, p.b_step, p.b_bytes, p.b_box, p.stage_bytes, p.ostride, p.hos, p.wos,
                       p.m64, p.ncw, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 48; i++) out[i] = v[i];
    return LVG_OK;
}

// the epilogue of that launch (host arithmetic only; tests/test_conv_epilogue_host.py checks it against the tiling)
extern "C" int lvg_convnd_epilogue_plan(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                        int pad_t, int pad_h, int pad_w, int stride, int* out, int out_len)
{
    LVG_REQUIRE(out && out_len >= 4, "convnd_epilogue_plan: out must hold 4 ints");
    int plan[48];
    const int rc = lvg_convnd_plan(mode, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, plan, 48);
    if (rc) return rc;
    for (int i = 0; i < out_len; i++) out[i] = 0;
    if (plan[47]) { out[0] = -1; return LVG_OK; }
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    IgemmParams p;
    const int prc = plan_igemm(mode == 0 ? fprop_job(sh, nullptr, nullptr, nullptr) : dgrad_job(sh, nullptr, nullptr, nullptr), p);
    if (prc) return prc;
    out[0] = p.pair_store;
    out[1] = p.stages;
    out[2] = igemm_smem_bytes(p);
    out[3] = kMapCols * (int)sizeof(int2);
    return LVG_OK;
}

// the tiling lvg_convnd_wgrad would launch with (host arithmetic only; tests/test_wgrad_emul.py replays it on the CPU, tools print it)
extern "C" int lvg_convnd_wgrad_plan(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                                     int pad_h, int pad_w, int* out, int out_len)
{
    LVG_REQUIRE(out && out_len >= 32, "convnd_wgrad_plan: out must hold 32 ints");
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!sh.wgrad_ok()) {
        set_error("convnd_wgrad_plan: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    const WgradPlan q = wgrad_plan(sh);
    const int v[32] = {q.split, q.cpad_a, q.cpad_b, q.nt, q.ntiles, q.mt, q.nsplit, q.ablk, q.khc, q.nseg, q.ps, q.rh, q.stages, q.a_stage, q.b_stage,
                       q.stage_bytes, q.tail_bytes, (int)q.smem, q.seg_w[0], q.seg_w[1], q.seg_w[2], q.seg_w[3], q.seg_x0[0], q.seg_x0[1], q.seg_x0[2],
                       q.seg_x0[3], 0, q.mrows, 0, 0, 0, 0};
    for (int i = 0; i < 32; i++) out[i] = v[i];
    return LVG_OK;
}

extern "C" int64_t lvg_convnd_backward_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                                 int pad_t, int pad_h, int pad_w)
{
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!sh.wgrad_ok()) return -1;
    // the engine's backward, or lvg_convnd_dgrad on a pointwise route followed by lvg_convnd_wgrad
    return std::max(backward_workspace(sh), pw_tc_workspace(dtype, cout, cin));
}

extern "C" int lvg_convnd_backward(const void* x, const void* dy, const void* w, void* dx, void* dw, int dtype, int n, int groups, int cin, int cout,
                                   int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, void* workspace,
                                   int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && dy && w && dx && dw, "convnd_backward: x, dy, w, dx, dw must not be NULL");
    LVG_REQUIRE(workspace && aligned16(workspace), "convnd_backward: workspace must be 16-byte aligned and not NULL");
    const ConvShape sh = {dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride};
    // the pointwise kernels read dy as it is: the two entry points one after the other
    if (!sh.wgrad_ok() || !sh.dgrad_ok() || lvg_convnd_route(1, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, 0) != 0) {
        const int rc = lvg_convnd_dgrad(dy, w, dx, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, workspace,
                                        workspace_bytes, stream);
        if (rc) return rc;
        return lvg_convnd_wgrad(x, dy, dw, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, workspace, workspace_bytes,
                                stream);
    }
    cudaStream_t s = (cudaStream_t)stream;
    Backward b;
    const int rc = backward_dgrad(sh, dy, nullptr, w, dx, workspace, workspace_bytes, s, b);
    if (rc) return rc;
    return backward_wgrad(sh, b, x, dy, nullptr, dw, nullptr, nullptr, s);
}
