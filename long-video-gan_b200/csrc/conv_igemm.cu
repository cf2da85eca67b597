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

#include <algorithm>
#include <cuda.h>
#include <stdlib.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"
#include "sres_cond.cuh"

namespace lvg {
// conv_pointwise.cu: streaming fp32 kernels for 1x1x1 convolutions with few channels (HBM-bound; the engine would re-tile and pad)
bool pw_supported(int dtype, int groups, int cin, int cout, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, int64_t P);
int pw_conv(const float* x, const float* w, float* y, int n, int cin, int cout, int64_t P, int64_t w_sco, int64_t w_sci, cudaStream_t s);
// conv_pw_tc.cu: every other 1x1x1 forward / input gradient on wgmma, straight from the NC(T)HW tensors (no re-tiling)
bool pw_tc_supported(int dtype, int groups, int cin, int cout, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, int64_t P);
int pw_tc_conv(const void* x, const void* w, void* y, int dtype, int n, int ck, int cm, int64_t P, int64_t w_sm, int64_t w_sk, void* workspace,
               int64_t workspace_bytes, cudaStream_t s, const void* res = nullptr, float rscale = 1.f);
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

struct IgemmParams {
    const unsigned char* wp;     // packed weights [wgroups][mt][kc][taps_all][a_img]
    void* y;
    const float* bias;           // per output channel (group-local index g*cout + co), or nullptr
    int act;                     // 0 = none, 1 = (x + b) * gain clamped, 2 = lrelu(x + b, alpha) * gain clamped
    float alpha, gain, clamp;    // clamp < 0: none
    int out_f32;
    int bf16;                    // operands are bf16 (split fp32) instead of fp16
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
    int64_t total_tiles;         // tiles_x * tiles_y * tiles_t * mt * instances
    int ks;                      // k-steps per stage (> 1 only when kt == 1)
    int stages;
    int a_resident;              // the ring length is a multiple of the stages per tile and every tile of the launch uses the same weights:
                                 // slot s always holds the same weight images -- they are fetched for the first `stages` iterations only
    int a_stage, b_step, b_bytes, b_box, stage_bytes;    // bytes: A per stage, B stride per k-step / per pair of blocks, TMA payload of a pair, whole stage
    int64_t y_cs;                // output channel stride (= to*hos*wos)
    int ostride, hos, wos;       // output decimation (strided convolution): only rows / columns divisible by ostride are stored
    const float* out_scale;      // per-(instance, output channel, output frame) factor [inst][cout][to] on the accumulator, or nullptr
};

// ------------------------------------------------------------------------------------------------ re-tiling passes

__device__ __forceinline__ unsigned short bf16_bits(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float bf16_val(unsigned short b) { return __uint_as_float((uint32_t)b << 16); }

// NC(T)HW -> X8. One thread = one pixel of one channel block: 8 strided reads (coalesced across the warp), one or two
// 16-byte writes. SPLIT: fp32 in, bf16 hi blocks [0, cblk) and lo blocks [cblk, 2 cblk) out.
// Dilation (gradients of strided convolutions): input pixel (t, i, j) of an ih x iw image lands at (t, i*dil, j*dil) of
// the oh x ow output image, which the caller has zeroed.
// `scale` (modulated convolutions): every element is multiplied by scale[instance][channel][frame] in fp32 before it is
// rounded to fp16 / split into bf16 halves; nullptr = the elements are copied as they are.
struct PackGeom { int64_t thw_in, thw_out; int ih, iw, oh, ow, dil; const float* scale; };

template <class TIn, bool SPLIT, bool SCALE>
__global__ void __launch_bounds__(256) conv_pack_act_kernel(const TIn* __restrict__ x, uint4* __restrict__ y, int64_t inst, int c,
                                                             int cblk, PackGeom gm)
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
            if constexpr (SCALE) {
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
                if constexpr (SCALE) { if (c0 + j < c) f *= __ldg(sc + j * frames); }
                hi[j] = bf16_bits(f);
                lo[j] = bf16_bits(f - bf16_val(hi[j]));
            }
            y[((int64_t)in * nblk + blk) * gm.thw_out + po] = *reinterpret_cast<const uint4*>(hi);
            y[((int64_t)in * nblk + cblk + blk) * gm.thw_out + po] = *reinterpret_cast<const uint4*>(lo);
        }
    }
}

// launches the re-tiling of one activation tensor (zeroing the target first when it is dilated)
int pack_act(const void* x, void* x8, int split, int64_t inst, int c, int cblk, int t, int ih, int iw, int oh, int ow, int dil, cudaStream_t s,
             const float* scale = nullptr)
{
    PackGeom gm;
    gm.thw_in = (int64_t)t * ih * iw; gm.thw_out = (int64_t)t * oh * ow; gm.ih = ih; gm.iw = iw; gm.oh = oh; gm.ow = ow; gm.dil = dil;
    gm.scale = scale;
    if (dil > 1) LVG_CUDA(cudaMemsetAsync(x8, 0, (size_t)(inst * (split ? 2 : 1) * cblk * gm.thw_out * 16), s));
    const int64_t total = inst * cblk * gm.thw_in;
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 64;
    if (blocks > cap) blocks = cap;
    // (the scaled variants are separate instantiations: the unscaled re-tiling stays the plain copy it was)
    if (split && scale) conv_pack_act_kernel<float, true, true><<<(unsigned)blocks, 256, 0, s>>>((const float*)x, (uint4*)x8, inst, c, cblk, gm);
    else if (split) conv_pack_act_kernel<float, true, false><<<(unsigned)blocks, 256, 0, s>>>((const float*)x, (uint4*)x8, inst, c, cblk, gm);
    else if (scale) conv_pack_act_kernel<__half, false, true><<<(unsigned)blocks, 256, 0, s>>>((const __half*)x, (uint4*)x8, inst, c, cblk, gm);
    else conv_pack_act_kernel<__half, false, false><<<(unsigned)blocks, 256, 0, s>>>((const __half*)x, (uint4*)x8, inst, c, cblk, gm);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

// upfirdn2d(x, f, padding = [2, 2, 2, 2]) (up 1, down 1) with a rank-1 4 x 4 filter f = outer(fy, fx), written straight
// into X8 of the filtered (h + 1) x (w + 1) image: the FIR of conv2d_resample's down-sampling 3x3 path fused into the
// re-tiling, so the filtered image never exists in NCHW. One CTA = one 8-channel block of one sample and a 32 x 8 tile of
// filtered pixels: the (8 + 3) x (32 + 3) input window of the 8 channels goes to shared memory once (zeros outside the
// image and past the last channel), a pass along y and one along x (fp32, taps in order) leave 8 values per thread, and
// the thread writes its pixel of the block as one 16-byte store (SPLIT: the bf16 hi and lo halves, one store each).
// gx / gy: the taps oriented for correlation (mirrored unless flip, as upfirdn2d orients them).
constexpr int kFirTX = 32, kFirTY = 8, kFirPitch = kFirTX + 4;

template <class TIn, bool SPLIT>
__global__ void __launch_bounds__(256) conv_pack_fir4_kernel(const TIn* __restrict__ x, uint4* __restrict__ y, int c, int cblk, int h, int w,
                                                              const float* __restrict__ fx, const float* __restrict__ fy, int flip)
{
    __shared__ float s_in[8][kFirTY + 3][kFirPitch];
    __shared__ float s_mid[8][kFirTY][kFirPitch];
    const int ho = h + 1, wo = w + 1;
    const int ox0 = blockIdx.x * kFirTX, oy0 = blockIdx.y * kFirTY;
    const int blk = (int)(blockIdx.z % cblk);
    const int64_t in = blockIdx.z / cblk;
    const int c0 = blk * 8;
    float gx[4], gy[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        gx[k] = __ldg(fx + (flip ? k : 3 - k));
        gy[k] = __ldg(fy + (flip ? k : 3 - k));
    }
    const TIn* xs = x + ((int64_t)in * c + c0) * h * w;
    for (int i = threadIdx.x; i < 8 * (kFirTY + 3) * (kFirTX + 3); i += 256) {
        const int col = i % (kFirTX + 3), r = (i / (kFirTX + 3)) % (kFirTY + 3), ch = i / ((kFirTX + 3) * (kFirTY + 3));
        const int iy = oy0 + r - 2, ix = ox0 + col - 2;
        float v = 0.f;
        if (c0 + ch < c && iy >= 0 && iy < h && ix >= 0 && ix < w) {
            if constexpr (SPLIT) v = __ldg(reinterpret_cast<const float*>(xs) + ((int64_t)ch * h + iy) * w + ix);
            else v = __half2float(__ldg(reinterpret_cast<const __half*>(xs) + ((int64_t)ch * h + iy) * w + ix));
        }
        s_in[ch][r][col] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * kFirTY * (kFirTX + 3); i += 256) {
        const int col = i % (kFirTX + 3), r = (i / (kFirTX + 3)) % kFirTY, ch = i / ((kFirTX + 3) * kFirTY);
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < 4; k++) v = fmaf(gy[k], s_in[ch][r + k][col], v);
        s_mid[ch][r][col] = v;
    }
    __syncthreads();
    const int tx = threadIdx.x % kFirTX, ty = threadIdx.x / kFirTX;
    const int oy = oy0 + ty, ox = ox0 + tx;
    if (oy >= ho || ox >= wo) return;
    float v[8];
#pragma unroll
    for (int ch = 0; ch < 8; ch++) {
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < 4; k++) a = fmaf(gx[k], s_mid[ch][ty][tx + k], a);
        v[ch] = a;
    }
    const int64_t plane = (int64_t)ho * wo, off = (int64_t)oy * wo + ox;
    if constexpr (!SPLIT) {
        alignas(16) __half o[8];
#pragma unroll
        for (int ch = 0; ch < 8; ch++) o[ch] = __float2half_rn(v[ch]);
        y[(in * cblk + blk) * plane + off] = *reinterpret_cast<const uint4*>(o);
    } else {
        alignas(16) unsigned short hi[8], lo[8];
#pragma unroll
        for (int ch = 0; ch < 8; ch++) {
            hi[ch] = bf16_bits(v[ch]);
            lo[ch] = bf16_bits(v[ch] - bf16_val(hi[ch]));
        }
        y[(in * 2 * cblk + blk) * plane + off] = *reinterpret_cast<const uint4*>(hi);
        y[(in * 2 * cblk + cblk + blk) * plane + off] = *reinterpret_cast<const uint4*>(lo);
    }
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

struct TileCoord { int ox0, oy0, t0, mti, inst; };

__device__ __forceinline__ TileCoord decode_tile(const IgemmParams& p, int64_t L)
{
    TileCoord c;
    int64_t r = L;
    c.ox0 = (int)(r % p.tiles_x) * p.wt; r /= p.tiles_x;
    c.oy0 = (int)(r % p.tiles_y) * p.th; r /= p.tiles_y;
    c.t0 = (int)(r % p.tiles_t) * p.tt; r /= p.tiles_t;
    c.mti = (int)(r % p.mt);
    c.inst = (int)(r / p.mt);
    return c;
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
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);

    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);     // warpgroup index, warp-uniform to the compiler
    const int taps2 = p.kh * p.kw;
    const int kchunks = (p.kc + p.ks - 1) / p.ks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        if (warp == 0 && elect_one()) {
            int it = 0;
            for (int64_t L = blockIdx.x; L < p.total_tiles; L += gridDim.x) {
                const TileCoord c = decode_tile(p, L);
                const unsigned char* wpg = p.wp + (((int64_t)(c.inst % p.wgroups) * p.mt + c.mti) * p.kc) * (int64_t)(p.kt * taps2) * (p.nimg * p.a_img);
                const int blk0 = c.inst * p.nblk;
                for (int kt = 0; kt < p.kt; kt++) {
                    for (int kcix = 0; kcix < kchunks; kcix++, it++) {
                        const int s = it % p.stages;
                        if (it >= p.stages) mbar_wait(&empty_bar[s], (uint32_t)((it / p.stages - 1) & 1));
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
        int it = 0;
        for (int64_t L = blockIdx.x; L < p.total_tiles; L += gridDim.x) {
            const TileCoord c = decode_tile(p, L);
            float acc[NW / 2];
#pragma unroll
            for (int i = 0; i < NW / 2; i++) acc[i] = 0.f;
            int prev = -1;
            for (int kt = 0; kt < p.kt; kt++) {
                for (int kcix = 0; kcix < kchunks; kcix++, it++) {
                    const int s = it % p.stages;
                    mbar_wait(&full_bar[s], (uint32_t)((it / p.stages) & 1));
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
            // r and r + 8 (conv_pack_w_kernel's row order -> channel) and column pairs col0 + 8 j + 2 (lane % 4).
            const int per = m_rows_per_quadrant(p.cout - c.mti * kBM);
            int64_t chbase[2];
            float bias[2];
            bool rok[2];
            const float* osc[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row = wq * 16 + lane / 4 + 8 * h;
                const int ch = p.m64 ? row : m_channel_of_row(cw * 64 + row, per);
                const int co = c.mti * kBM + ch;
                rok[h] = ch < kBM && co < p.cout;
                bias[h] = (p.bias != nullptr && rok[h]) ? __ldg(p.bias + (int64_t)(c.inst % p.wgroups) * p.cout + co) : 0.f;
                chbase[h] = ((int64_t)c.inst * p.cout + co) * p.y_cs;
                osc[h] = OSCALE ? p.out_scale + ((int64_t)c.inst * p.cout + co) * p.to : nullptr;
            }
#pragma unroll
            for (int j = 0; j < NW / 8; j++) {
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    // accumulator column -> (frame, row, col) of the tile
                    const int n = col0 + j * 8 + 2 * (lane % 4) + e;
                    const int f = n / p.frame_px, rem = n - f * p.frame_px;
                    const int r = rem / p.wtb, cc = rem - r * p.wtb;
                    const int ot = c.t0 + f, oy = c.oy0 + r, ox = c.ox0 + cc;
                    bool ok = n < p.ncols && f < p.tt && r < p.th && cc < p.wt && ot < p.to && oy < p.ho && ox < p.wo;
                    int64_t off;
                    if (p.ostride == 1) {
                        off = ((int64_t)ot * p.ho + oy) * p.wo + ox;
                    } else {
                        ok = ok && (oy % p.ostride == 0) && (ox % p.ostride == 0);
                        off = ((int64_t)ot * p.hos + oy / p.ostride) * p.wos + ox / p.ostride;
                    }
                    if (!ok) continue;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        if (!rok[h]) continue;
                        float v = acc[4 * j + 2 * h + e];
                        if constexpr (OSCALE) v *= __ldg(osc[h] + ot);
                        if (p.act) {
                            v += bias[h];
                            if (p.act == 2) v = v < 0.f ? v * p.alpha : v;
                            v *= p.gain;
                            if (p.clamp >= 0.f) v = fminf(fmaxf(v, -p.clamp), p.clamp);
                        }
                        if (p.out_f32) reinterpret_cast<float*>(p.y)[chbase[h] + off] = v;
                        else reinterpret_cast<__half*>(p.y)[chbase[h] + off] = __float2half_rn(v);
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

inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

inline int env_flag(const char* name, int dflt)
{
    const char* e = getenv(name);
    return e ? atoi(e) : dflt;
}

struct Geometry {
    int cpad, cblk, nblk, nimg, kc, mt;
    int m64, a_img;              // 64-row mode, bytes of one weight image
    int64_t act_bytes, w_bytes;
};

// K-side geometry for `ck` contraction channels and `cm` output channels per group
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

// shared driver of fprop and dgrad: `x` has `ck` channels per group, `y` gets `cm`; logical A[m][k][tap] = w[g*gs + m*sm + k*sk + tap']
// `dil` > 1: x is given as an xin_h x xin_w image that is placed on every dil-th pixel of the h x wd grid (input gradient of
// a strided convolution); `ostride` > 1: only every ostride-th output row / column is stored (strided forward convolution).
// lvg_convnd_plan: run_igemm stops after its tile selection (pure host arithmetic, no CUDA call) and hands the parameters out
thread_local IgemmParams* g_plan_only = nullptr;

int run_igemm(const void* x, const void* w, void* y, int dtype, int n, int groups, int ck, int cm, int t, int h, int wd, int kt, int kh,
              int kw, int pad_t, int pad_h, int pad_w, int64_t w_gs, int64_t w_sm, int64_t w_sk, int flip, const float* bias, int act,
              float alpha, float gain, float clamp, int xin_h, int xin_w, int dil, int ostride, const unsigned char* x8_pre, void* workspace,
              int64_t workspace_bytes, cudaStream_t s, const float* in_scale = nullptr, const float* out_scale = nullptr)
{
    // `in_scale` [n][ck][t] multiplies x while it is re-tiled (not with x8_pre: the caller re-tiled it), `out_scale`
    // [n][cm][to] the accumulators in the epilogue (groups == 1: instance = sample)
    // `x8_pre` != nullptr: x is already re-tiled there (lvg_convnd_backward shares dy8 with the weight gradient); the workspace
    // then only holds the packed weights
    const int split = dtype == LVG_F32 ? 1 : 0;
    const int taps = kt * kh * kw;
    const int64_t inst = (int64_t)n * groups;
    const int64_t thw = (int64_t)t * h * wd;
    const Geometry g = geometry(split, inst, groups, ck, cm, thw, taps);
    const bool plan_only = g_plan_only != nullptr;
    LVG_REQUIRE(plan_only || (workspace && workspace_bytes >= (x8_pre ? 0 : g.act_bytes) + g.w_bytes + 256), "convnd: workspace too small");
    LVG_REQUIRE(plan_only || aligned16(workspace), "convnd: workspace must be 16-byte aligned");
    LVG_REQUIRE(inst * g.nblk < (1ll << 31), "convnd: too many channel blocks for a tensor map");
    EncodeTiledFn enc = plan_only ? nullptr : encode_fn();
    LVG_REQUIRE(plan_only || enc != nullptr, "convnd: cuTensorMapEncodeTiled is not available from this driver");

    unsigned char* wp = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* x8 = x8_pre ? const_cast<unsigned char*>(x8_pre) : wp + ((g.w_bytes + 127) / 128) * 128;

    IgemmParams p;
    memset(&p, 0, sizeof(p));
    p.wp = wp; p.y = y; p.bias = bias; p.act = act; p.alpha = alpha; p.gain = gain; p.clamp = clamp; p.out_scale = out_scale;
    p.out_f32 = split; p.bf16 = split;
    p.wgroups = groups; p.cout = cm; p.mt = g.mt; p.kc = g.kc; p.nblk = g.nblk;
    p.nimg = g.nimg; p.lo_blk = g.cblk;
    p.m64 = g.m64; p.a_img = g.a_img;
    p.to = t + 2 * pad_t - kt + 1; p.ho = h + 2 * pad_h - kh + 1; p.wo = wd + 2 * pad_w - kw + 1;
    LVG_REQUIRE(p.to >= 1 && p.ho >= 1 && p.wo >= 1, "convnd: empty output");
    p.kt = kt; p.kh = kh; p.kw = kw; p.pad_t = pad_t; p.pad_h = pad_h; p.pad_w = pad_w;
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
        if (groups == 1 && g.mt == 1 && period <= p.stages && env_flag("LVG_CONV_RESIDENT_W", 1)) {
            p.stages = p.stages / period * period;
            p.a_resident = 1;
        }
    }
    p.y_cs = (int64_t)p.to * p.hos * p.wos;
    p.total_tiles = (int64_t)p.tiles_x * p.tiles_y * p.tiles_t * g.mt * inst;

    if (plan_only) { *g_plan_only = p; return LVG_OK; }

    // re-tile the operands
    {
        const int rc = x8_pre ? LVG_OK : pack_act(x, x8, split, inst, ck, g.cblk, t, xin_h, xin_w, h, wd, dil, s, in_scale);
        if (rc) return rc;
        const int64_t wblocks = (int64_t)groups * g.mt * g.kc;
        LVG_REQUIRE(wblocks < (1ll << 31), "convnd: too many weight tiles");
        // rows of m per pass: <= ~64 KB of staging (16 * rows * taps elements either way)
        const int es = split ? 4 : 2;
        const int img_rows = g.m64 ? 64 : kBM;
        int rpp = (int)((64 * 1024) / (16 * taps * es + 16)) / 8 * 8;
        if (rpp > img_rows) rpp = img_rows;
        if (rpp < 8) rpp = 8;
        const bool mrows = w_sk < w_sm;
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
            conv_pack_w_kernel<float, true><<<wgrid, 256, wsm, s>>>((const float*)w, wp, cm, ck, g.cpad, taps, w_gs, w_sm, w_sk, flip, g.mt, g.kc, rpp, rows_per_cta, img_rows);
        } else {
            LVG_CUDA(cudaFuncSetAttribute(conv_pack_w_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm));
            conv_pack_w_kernel<__half, false><<<wgrid, 256, wsm, s>>>((const __half*)w, wp, cm, ck, g.cpad, taps, w_gs, w_sm, w_sk, flip, g.mt, g.kc, rpp, rows_per_cta, img_rows);
        }
        LVG_LAUNCH_CHECK();
    }

    // tensor map over X8 as 8-byte elements: (2 W, H, T, instance * block)
    CUtensorMap tm;
    {
        const int rc = encode_map(&tm, x8, wd, h, t, inst * g.nblk, wd, (int64_t)h * wd, thw, p.wtb, p.thb, p.tt, 2);
        if (rc) return rc;
    }
    const size_t smem = (size_t)p.stages * p.stage_bytes + 128;
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
    void (*kern)(const CUtensorMap, const IgemmParams) = kerns[out_scale != nullptr][split][p.ncw / 16 - 1];
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const char* cta_env = getenv("LVG_CONV_CTAS");          // experiments: fewer persistent CTAs than SMs
    const int max_ctas = cta_env ? atoi(cta_env) : num_sms();
    int64_t ctas = p.total_tiles < max_ctas ? p.total_tiles : max_ctas;
    kern<<<(unsigned)ctas, kIgemmThreads, smem, s>>>(tm, p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

bool nd_supported(int dtype, int kt, int kh, int kw)
{
    return (dtype == LVG_F16 || dtype == LVG_F32) && kt >= 1 && kh >= 1 && kw >= 1 && kh * kw <= 9 && kt <= 7;
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_convnd_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                        int pad_t, int pad_h, int pad_w)
{
    if (!nd_supported(dtype, kt, kh, kw) || n < 1 || groups < 1) return -1;
    const int split = dtype == LVG_F32;
    const int taps = kt * kh * kw;
    const int64_t inst = (int64_t)n * groups;
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    if (to < 1 || ho < 1 || wo < 1) return -1;
    const Geometry a = geometry(split, inst, groups, cin, cout, (int64_t)t * h * wd, taps);        // fprop
    const Geometry b = geometry(split, inst, groups, cout, cin, (int64_t)to * ho * wo, taps);      // dgrad
    const int64_t fa = a.act_bytes + a.w_bytes, fb = b.act_bytes + b.w_bytes;
    return (fa > fb ? fa : fb) + 1024;
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
    if (!nd_supported(dtype, kt, kh, kw) || n < 1 || pad_t < 0 || pad_h < 0 || pad_w < 0 || stride < 1 || stride > 4) {
        set_error("convnd_fprop: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    const int taps = kt * kh * kw;
    return run_igemm(x, w, y, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, (int64_t)cout * cin * taps,
                     (int64_t)cin * taps, taps, 0, bias, act, alpha, gain, clamp, h, wd, 1, stride, nullptr, workspace, workspace_bytes,
                     (cudaStream_t)stream);
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
    if (!nd_supported(dtype, kt, kh, kw) || n < 1 || pad_t < 0 || pad_h < 0 || pad_w < 0 || pad_t > kt - 1 || pad_h > kh - 1 || pad_w > kw - 1 ||
        stride < 1 || stride > 4) {
        set_error("convnd_dgrad: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    // dx = correlation of dy (to x ho x wo, cout channels; for a strided convolution: dy spread over every stride-th pixel of
    // that grid) with the channel-transposed, mirrored weights, padding k-1-pad
    const int taps = kt * kh * kw;
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    const int hos = (ho - 1) / stride + 1, wos = (wo - 1) / stride + 1;
    return run_igemm(dy, w, dx, dtype, n, groups, cout, cin, to, ho, wo, kt, kh, kw, kt - 1 - pad_t, kh - 1 - pad_h, kw - 1 - pad_w,
                     (int64_t)cout * cin * taps, taps, (int64_t)cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, hos, wos, stride, 1, nullptr, workspace,
                     workspace_bytes, (cudaStream_t)stream);
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

struct WgradPlan {
    int split, cpad_a, cpad_b, nt, ntiles, mt, nsplit;
    int ablk, khc, mrows;
    int nseg, seg_w[4], seg_x0[4], ps, rh, stages;
    int a_stage, b_stage, stage_bytes, tail_bytes;
    size_t smem;
    int64_t a_bytes, b_bytes, part_bytes, dw_elems;
};

// channel padding of the dy8 operand of the weight gradient. cout < 128: only the channel blocks that exist (the same
// tensor the input gradient reads, so one re-tiling pass serves both; the remaining rows of the 128-row MMA read whatever
// follows in shared memory and are never stored -- rows of D depend on the same rows of A only). Otherwise whole m-tiles.
inline int wgrad_cpad_a(int cout) { return (cout < kBM && env_flag("LVG_WGRAD_COMPACT", 1)) ? round_up(cout, 16) : round_up(cout, kBM); }

WgradPlan wgrad_plan(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int to, int ho, int wo, int kt, int kh, int kw,
                     bool fold = true)
{
    WgradPlan q;
    q.split = dtype == LVG_F32;
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
    const int64_t inst = (int64_t)n * groups;
    q.a_bytes = inst * nop * (q.cpad_a / 8) * (int64_t)to * ho * wo * 16;
    q.b_bytes = inst * nop * (q.cpad_b / 8) * (int64_t)t * h * wd * 16;
    q.dw_elems = (int64_t)groups * cout * cin * kt * kh * kw;
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
    if (q.khc > 1 && q.smem > 227 * 1024) return wgrad_plan(dtype, n, groups, cin, cout, t, h, wd, to, ho, wo, kt, kh, kw, false);
    // Split the pixel range over `nsplit` CTAs per output tile. One CTA per SM is resident, so the kernel runs in waves of
    // num_sms CTAs: choose the split that minimises waves x (stages per CTA + a fixed per-CTA cost of ~4 stages: clearing
    // shared memory, the register -> global epilogue) -- e.g. with 132 SMs and 3 output tiles: 44 splits = 132 CTAs = one
    // wave instead of 64 splits = 192 CTAs = two waves. Partial sums are capped at 256 MB.
    const int64_t ctas = (int64_t)q.ntiles * (kh / q.khc) * kt * q.mt * groups;
    const int64_t stages = (int64_t)n * to * q.nseg * ((ho + q.rh - 1) / q.rh);
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

// the weight-gradient launch; `dy8_pre` != nullptr: dy is already re-tiled (the tensor the input gradient of the same call read)
int run_wgrad(const void* x, const void* dy, void* dw, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh,
              int kw, int pad_t, int pad_h, int pad_w, int stride, const unsigned char* dy8_pre, void* workspace, int64_t workspace_bytes,
              cudaStream_t s, const float* x_scale = nullptr, const float* dy_scale = nullptr, const unsigned char* x8_pre = nullptr)
{
    // `x8_pre` != nullptr: x is already re-tiled there, with cpad_b / 8 blocks (conv_pack_fir4_kernel: the filtered image of
    // a super-res discriminator block); x is not read
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    const WgradPlan q = wgrad_plan(dtype, n, groups, cin, cout, t, h, wd, to, ho, wo, kt, kh, kw);
    const int64_t a_room = dy8_pre ? 0 : ((q.a_bytes + 255) / 256) * 256;
    LVG_REQUIRE(workspace && workspace_bytes >= a_room + q.b_bytes + q.part_bytes + 768, "convnd_wgrad: workspace too small");
    LVG_REQUIRE(aligned16(workspace), "convnd_wgrad: workspace must be 16-byte aligned");
    LVG_REQUIRE(groups <= 65535 && q.mt <= 65535, "convnd_wgrad: too many groups / channel tiles");
    const int64_t inst = (int64_t)n * groups;
    unsigned char* x8 = x8_pre ? const_cast<unsigned char*>(x8_pre) : reinterpret_cast<unsigned char*>(workspace) + a_room;
    unsigned char* dy8 = dy8_pre ? const_cast<unsigned char*>(dy8_pre) : reinterpret_cast<unsigned char*>(workspace);
    float* part = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + a_room + ((q.b_bytes + 255) / 256) * 256);
    const int64_t thw_a = (int64_t)to * ho * wo, thw_b = (int64_t)t * h * wd;
    {
        // dy of a strided convolution is spread over every stride-th pixel of the stride-1 output grid (zeros between)
        int rc = dy8_pre ? LVG_OK : pack_act(dy, dy8, q.split, inst, cout, q.cpad_a / 8, to, (ho - 1) / stride + 1, (wo - 1) / stride + 1, ho, wo, stride, s,
                                             dy_scale);
        if (rc) return rc;
        rc = x8_pre ? LVG_OK : pack_act(x, x8, q.split, inst, cin, q.cpad_b / 8, t, h, wd, h, wd, 1, s, x_scale);   // x_scale [n][cin][t]: x is modulated
        if (rc) return rc;
    }
    WgradV2Params p;
    memset(&p, 0, sizeof(p));
    p.out_f32 = q.split; p.bf16 = q.split; p.split = q.split;
    p.n = n; p.groups = groups; p.cin = cin; p.cout = cout; p.to = to; p.ho = ho;
    p.kt = kt; p.kh = kh; p.kw = kw; p.pad_t = pad_t; p.pad_h = pad_h; p.pad_w = pad_w;
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
        const int rc = encode_map(&maps.b, x8, wd, h, t, inst * p.nblk_b, wd, (int64_t)h * wd, thw_b, p.ps[0], p.rh + q.khc - 1, 1, q.nt / 8);
        if (rc) return rc;
    }
    void (*const kern)(const WgradMaps, const WgradV2Params) = wgrad_kernel(q.split, q.khc * kw, q.nt);
    LVG_REQUIRE(kern != nullptr, "convnd_wgrad: no kernel for %d taps x %d columns (split %d)", q.khc * kw, q.nt, q.split);
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((unsigned)(q.ntiles * kt * (kh / q.khc) * q.nsplit), (unsigned)q.mt, (unsigned)groups);
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

bool wgrad_in_envelope(int dtype, int n, int groups, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride)
{
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    return nd_supported(dtype, kt, kh, kw) && n >= 1 && groups >= 1 && kw <= 3 && pad_t >= 0 && pad_h >= 0 && pad_w >= 0 && to >= 1 && ho >= 1 &&
           wo >= 1 && wo <= 4 * (128 - kw + 1) && stride >= 1 && stride <= 4;
}

}  // namespace
}  // namespace lvg

extern "C" int64_t lvg_convnd_wgrad_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                              int pad_t, int pad_h, int pad_w)
{
    if (!wgrad_in_envelope(dtype, n, groups, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1)) return -1;
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    const WgradPlan q = wgrad_plan(dtype, n, groups, cin, cout, t, h, wd, to, ho, wo, kt, kh, kw);
    return q.a_bytes + q.b_bytes + q.part_bytes + 1024;
}

extern "C" int lvg_convnd_wgrad(const void* x, const void* dy, void* dw, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                                int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, void* workspace, int64_t workspace_bytes,
                                void* stream)
{
    LVG_REQUIRE(x && dy && dw, "convnd_wgrad: x, dy, dw must not be NULL");
    if (!wgrad_in_envelope(dtype, n, groups, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride)) {
        set_error("convnd_wgrad: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    return run_wgrad(x, dy, dw, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, nullptr, workspace, workspace_bytes,
                     (cudaStream_t)stream);
}

// which kernels a call takes (host arithmetic only): mode 0 forward (`epilogue` != 0: with a bias / activation / gain /
// clamp epilogue), 1 input gradient, 2 weight gradient -> 0 the engine, 1 the streaming SIMT kernels (conv_pointwise.cu),
// 2 the pointwise wgmma kernels (conv_pw_tc.cu); LVG_UNSUPPORTED outside the envelope. Tensors are taken to be 16-byte
// aligned (the pointwise wgmma route falls back to the engine for a misaligned one).
extern "C" int lvg_convnd_route(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                                int pad_h, int pad_w, int stride, int epilogue)
{
    if (mode < 0 || mode > 2 || n < 1 || groups < 1) return LVG_UNSUPPORTED;
    if (mode == 2) return wgrad_in_envelope(dtype, n, groups, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride) ? 0 : LVG_UNSUPPORTED;
    const int64_t P = (int64_t)t * h * wd;
    if (mode == 1 || !epilogue) {
        if (pw_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, P)) return 1;
        if (pw_tc_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, P)) return 2;
    }
    if (!nd_supported(dtype, kt, kh, kw) || pad_t < 0 || pad_h < 0 || pad_w < 0 || stride < 1 || stride > 4 ||
        (mode == 1 && (pad_t > kt - 1 || pad_h > kh - 1 || pad_w > kw - 1)))
        return LVG_UNSUPPORTED;
    return 0;
}

// the tiling lvg_convnd_fprop (mode 0) / lvg_convnd_dgrad (mode 1) would launch with, as ints (host arithmetic only;
// tests/test_igemm_emul.py replays the forward kernel's addressing with it on the CPU)
extern "C" int lvg_convnd_plan(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                               int pad_h, int pad_w, int stride, int* out, int out_len)
{
    LVG_REQUIRE(out && out_len >= 48, "convnd_plan: out must hold 48 ints");
    LVG_REQUIRE(mode == 0 || mode == 1, "convnd_plan: mode 0 (forward) or 1 (input gradient)");
    const int taps = kt * kh * kw;
    if (!nd_supported(dtype, kt, kh, kw) || n < 1 || groups < 1 || pad_t < 0 || pad_h < 0 || pad_w < 0 || stride < 1 || stride > 4 ||
        (mode == 1 && (pad_t > kt - 1 || pad_h > kh - 1 || pad_w > kw - 1))) {
        set_error("convnd_plan: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    for (int i = 0; i < out_len; i++) out[i] = 0;
    if (pw_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, (int64_t)t * h * wd)) { out[47] = 1; return LVG_OK; }
    IgemmParams p;
    memset(&p, 0, sizeof(p));
    void* dummy = reinterpret_cast<void*>(256);          // never dereferenced in plan-only mode
    g_plan_only = &p;
    int rc;
    if (mode == 0) {
        rc = run_igemm(dummy, dummy, dummy, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, (int64_t)cout * cin * taps,
                       (int64_t)cin * taps, taps, 0, nullptr, 0, 0.f, 1.f, -1.f, h, wd, 1, stride, nullptr, nullptr, 0, nullptr);
    } else {
        const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
        if (to < 1 || ho < 1 || wo < 1) { g_plan_only = nullptr; set_error("convnd_plan: empty output"); return LVG_UNSUPPORTED; }
        const int hos = (ho - 1) / stride + 1, wos = (wo - 1) / stride + 1;
        rc = run_igemm(dummy, dummy, dummy, dtype, n, groups, cout, cin, to, ho, wo, kt, kh, kw, kt - 1 - pad_t, kh - 1 - pad_h, kw - 1 - pad_w,
                       (int64_t)cout * cin * taps, taps, (int64_t)cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, hos, wos, stride, 1, nullptr, nullptr, 0,
                       nullptr);
    }
    g_plan_only = nullptr;
    if (rc) return rc;
    const int v[48] = {p.wgroups, p.cout, p.mt, p.kc, p.nblk, p.nimg, p.lo_blk, p.to, p.ho, p.wo, p.kt, p.kh, p.kw, p.pad_t, p.pad_h, p.pad_w,
                       p.tt, p.th, p.wt, p.wtb, p.thb, p.frame_px, p.ncols, p.tiles_x, p.tiles_y, p.tiles_t,
                       (int)p.total_tiles, p.ks, p.stages, p.a_resident, p.a_stage, p.b_step, p.b_bytes, p.b_box, p.stage_bytes, p.ostride, p.hos, p.wos,
                       p.m64, p.ncw, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 48; i++) out[i] = v[i];
    return LVG_OK;
}

// the tiling lvg_convnd_wgrad would launch with (host arithmetic only; tests/test_wgrad_emul.py replays it on the CPU, tools print it)
extern "C" int lvg_convnd_wgrad_plan(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                                     int pad_h, int pad_w, int* out, int out_len)
{
    LVG_REQUIRE(out && out_len >= 32, "convnd_wgrad_plan: out must hold 32 ints");
    if (!wgrad_in_envelope(dtype, n, groups, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1)) {
        set_error("convnd_wgrad_plan: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    const WgradPlan q = wgrad_plan(dtype, n, groups, cin, cout, t, h, wd, to, ho, wo, kt, kh, kw);
    const int v[32] = {q.split, q.cpad_a, q.cpad_b, q.nt, q.ntiles, q.mt, q.nsplit, q.ablk, q.khc, q.nseg, q.ps, q.rh, q.stages, q.a_stage, q.b_stage,
                       q.stage_bytes, q.tail_bytes, (int)q.smem, q.seg_w[0], q.seg_w[1], q.seg_w[2], q.seg_w[3], q.seg_x0[0], q.seg_x0[1], q.seg_x0[2],
                       q.seg_x0[3], 0, q.mrows, 0, 0, 0, 0};
    for (int i = 0; i < 32; i++) out[i] = v[i];
    return LVG_OK;
}

// ---- both gradients of one convolution call. dy is re-tiled ONCE: the input gradient (forward kernel on dy) and the weight
// gradient (dy as the M-side operand) read the same channel-block tensor whenever their paddings agree (cout < 128 or a
// multiple of 128: every layer of the networks); otherwise, and for the streaming 1x1x1 kernels, the two entry points above run
// one after the other. Workspace layout of the shared case: [dy8][packed weights of the input gradient][x8][partial sums].
namespace lvg {
namespace {
bool backward_shares_dy8(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h,
                         int pad_w, int stride)
{
    const int64_t P = (int64_t)t * h * wd;
    if (!env_flag("LVG_CONV_SHARED_DY8", 1)) return false;
    if (pw_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, P)) return false;
    if (pw_tc_supported(dtype, groups, cin, cout, kt, kh, kw, pad_t, pad_h, pad_w, stride, P)) return false;     // reads dy as it is
    return wgrad_cpad_a(cout) == round_up(cout, 16);
}
}  // namespace
}  // namespace lvg

extern "C" int64_t lvg_convnd_backward_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                                 int pad_t, int pad_h, int pad_w)
{
    const int64_t a = lvg_convnd_workspace(dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w);
    const int64_t b = lvg_convnd_wgrad_workspace(dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w);
    if (a < 0 || b < 0) return -1;
    // (the shared layout never needs more than the two separate ones together)
    return a + b + 1024;
}

extern "C" int lvg_convnd_backward(const void* x, const void* dy, const void* w, void* dx, void* dw, int dtype, int n, int groups, int cin, int cout,
                                   int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, void* workspace,
                                   int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && dy && w && dx && dw, "convnd_backward: x, dy, w, dx, dw must not be NULL");
    LVG_REQUIRE(workspace && aligned16(workspace), "convnd_backward: workspace must be 16-byte aligned and not NULL");
    const bool tc_ok = wgrad_in_envelope(dtype, n, groups, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride) && pad_t <= kt - 1 && pad_h <= kh - 1 &&
                       pad_w <= kw - 1;
    if (!tc_ok || !backward_shares_dy8(dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride)) {
        const int rc = lvg_convnd_dgrad(dy, w, dx, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, workspace,
                                        workspace_bytes, stream);
        if (rc) return rc;
        return lvg_convnd_wgrad(x, dy, dw, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, workspace, workspace_bytes,
                                stream);
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int split = dtype == LVG_F32 ? 1 : 0;
    const int taps = kt * kh * kw;
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    const int hos = (ho - 1) / stride + 1, wos = (wo - 1) / stride + 1;
    const int64_t inst = (int64_t)n * groups;
    const Geometry gd = geometry(split, inst, groups, cout, cin, (int64_t)to * ho * wo, taps);      // the input gradient's operands
    const int64_t dy8_room = ((gd.act_bytes + 255) / 256) * 256;
    const int64_t wp_room = ((gd.w_bytes + 255) / 256) * 256 + 256;
    LVG_REQUIRE(workspace_bytes >= dy8_room + wp_room, "convnd_backward: workspace too small");
    unsigned char* dy8 = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* rest = dy8 + dy8_room;
    int rc = pack_act(dy, dy8, split, inst, cout, gd.cblk, to, hos, wos, ho, wo, stride, s);
    if (rc) return rc;
    rc = run_igemm(dy, w, dx, dtype, n, groups, cout, cin, to, ho, wo, kt, kh, kw, kt - 1 - pad_t, kh - 1 - pad_h, kw - 1 - pad_w,
                   (int64_t)cout * cin * taps, taps, (int64_t)cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, hos, wos, stride, 1, dy8, rest, wp_room, s);
    if (rc) return rc;
    // (stream order: the weight gradient's re-tiling of x overwrites the packed weights only after the input gradient read them)
    return run_wgrad(x, dy, dw, dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride, dy8, rest,
                     workspace_bytes - dy8_room, s);
}

// ---- conv1 of a super-res discriminator block (conv2d_resample with down = 2, a 3x3 kernel and padding 1): the 4-tap FIR
// with padding 2 runs inside the re-tiling pass (conv_pack_fir4_kernel), the stride-2 convolution and its bias_act epilogue
// on the engine as lvg_convnd_fprop runs them. Workspace: [packed weights][X8 of the filtered image].
extern "C" int64_t lvg_sres_dblock_conv1_workspace(int dtype, int n, int cin, int cout, int h, int wd)
{
    if ((dtype != LVG_F16 && dtype != LVG_F32) || n < 1 || cin < 1 || cout < 1 || h < 2 || wd < 2) return -1;
    const int hf = h + 1, wf = wd + 1;
    const Geometry g = geometry(dtype == LVG_F32, n, 1, cin, cout, (int64_t)hf * wf, 9);
    if ((int64_t)n * g.cblk > 65535 || (int64_t)n * g.nblk >= (1ll << 31) || wf - 2 > 4 * (128 - 2)) return -1;
    return ((g.w_bytes + 256 + 255) / 256) * 256 + g.act_bytes + 256;
}

extern "C" int lvg_sres_dblock_conv1(const void* x, const float* fx, const float* fy, int flip, const void* w, const float* bias, void* y, int dtype,
                                     int n, int cin, int cout, int h, int wd, int act, float alpha, float gain, float clamp, void* workspace,
                                     int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && fx && fy && w && y, "sres_dblock_conv1: x, fx, fy, w, y must not be NULL");
    const int64_t need = lvg_sres_dblock_conv1_workspace(dtype, n, cin, cout, h, wd);
    if (need < 0) {
        set_error("sres_dblock_conv1: outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= need, "sres_dblock_conv1: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    const int split = dtype == LVG_F32;
    const int hf = h + 1, wf = wd + 1;
    const Geometry g = geometry(split, n, 1, cin, cout, (int64_t)hf * wf, 9);
    const int64_t wp_room = ((g.w_bytes + 256 + 255) / 256) * 256;
    unsigned char* x8 = reinterpret_cast<unsigned char*>(workspace) + wp_room;
    {
        const dim3 grid((unsigned)((wf + kFirTX - 1) / kFirTX), (unsigned)((hf + kFirTY - 1) / kFirTY), (unsigned)(n * g.cblk));
        if (split) conv_pack_fir4_kernel<float, true><<<grid, 256, 0, s>>>((const float*)x, (uint4*)x8, cin, g.cblk, h, wd, fx, fy, flip);
        else conv_pack_fir4_kernel<__half, false><<<grid, 256, 0, s>>>((const __half*)x, (uint4*)x8, cin, g.cblk, h, wd, fx, fy, flip);
        LVG_LAUNCH_CHECK();
    }
    return run_igemm(x8, w, y, dtype, n, 1, cin, cout, 1, hf, wf, 1, 3, 3, 0, 0, 0, (int64_t)cout * cin * 9, (int64_t)cin * 9, 9, 0, bias, act, alpha,
                     gain, clamp, hf, wf, 1, 2, x8, workspace, wp_room, s);
}

// ---- conv1's backward: dhf = the input gradient of the strided convolution (the filtered image's gradient, (h + 1) x (wd + 1),
// lvg_convnd_dgrad), and dw from the weight-gradient kernel with its B operand re-tiled straight from x by
// conv_pack_fir4_kernel (the filtered image is recomputed into X8, never into NCHW). Workspace: [X8 of the filtered image]
// [the larger of the two kernels' workspaces].
namespace lvg {
namespace {
int64_t conv1_bwd_x8_bytes(int dtype, int n, int cin, int cout, int h, int wd)
{
    const WgradPlan q = wgrad_plan(dtype, n, 1, cin, cout, 1, h + 1, wd + 1, 1, h - 1, wd - 1, 1, 3, 3);
    return ((q.b_bytes + 255) / 256) * 256;
}
}  // namespace
}  // namespace lvg

extern "C" int64_t lvg_sres_dblock_conv1_backward_workspace(int dtype, int n, int cin, int cout, int h, int wd)
{
    if (lvg_sres_dblock_conv1_workspace(dtype, n, cin, cout, h, wd) < 0) return -1;
    if (!wgrad_in_envelope(dtype, n, 1, 1, h + 1, wd + 1, 1, 3, 3, 0, 0, 0, 2)) return -1;
    const int64_t a = lvg_convnd_workspace(dtype, n, 1, cin, cout, 1, h + 1, wd + 1, 1, 3, 3, 0, 0, 0);
    const int64_t b = lvg_convnd_wgrad_workspace(dtype, n, 1, cin, cout, 1, h + 1, wd + 1, 1, 3, 3, 0, 0, 0);
    if (a < 0 || b < 0) return -1;
    return conv1_bwd_x8_bytes(dtype, n, cin, cout, h, wd) + (a > b ? a : b) + 1024;
}

extern "C" int lvg_sres_dblock_conv1_backward(const void* x, const float* fx, const float* fy, int flip, const void* dy, const void* w, void* dhf,
                                              void* dw, int dtype, int n, int cin, int cout, int h, int wd, void* workspace, int64_t workspace_bytes,
                                              void* stream)
{
    LVG_REQUIRE(x && fx && fy && dy && w && (dhf || dw), "sres_dblock_conv1_backward: x, fx, fy, dy, w and dhf or dw must not be NULL");
    const int64_t need = lvg_sres_dblock_conv1_backward_workspace(dtype, n, cin, cout, h, wd);
    if (need < 0) {
        set_error("sres_dblock_conv1_backward: outside the kernels' envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= need, "sres_dblock_conv1_backward: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    const int hf = h + 1, wf = wd + 1;
    const int64_t x8_room = conv1_bwd_x8_bytes(dtype, n, cin, cout, h, wd);
    unsigned char* x8 = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* rest = x8 + x8_room;
    const int64_t rest_bytes = workspace_bytes - x8_room;
    if (dhf) {
        const int rc = lvg_convnd_dgrad(dy, w, dhf, dtype, n, 1, cin, cout, 1, hf, wf, 1, 3, 3, 0, 0, 0, 2, rest, rest_bytes, stream);
        if (rc) return rc;
    }
    if (!dw) return LVG_OK;
    const WgradPlan q = wgrad_plan(dtype, n, 1, cin, cout, 1, hf, wf, 1, hf - 2, wf - 2, 1, 3, 3);
    const int cblk = q.cpad_b / 8;
    LVG_REQUIRE((int64_t)n * cblk <= 65535, "sres_dblock_conv1_backward: too many channel blocks");
    {
        const dim3 grid((unsigned)((wf + kFirTX - 1) / kFirTX), (unsigned)((hf + kFirTY - 1) / kFirTY), (unsigned)(n * cblk));
        if (q.split) conv_pack_fir4_kernel<float, true><<<grid, 256, 0, s>>>((const float*)x, (uint4*)x8, cin, cblk, h, wd, fx, fy, flip);
        else conv_pack_fir4_kernel<__half, false><<<grid, 256, 0, s>>>((const __half*)x, (uint4*)x8, cin, cblk, h, wd, fx, fy, flip);
        LVG_LAUNCH_CHECK();
    }
    return run_wgrad(nullptr, dy, dw, dtype, n, 1, cin, cout, 1, hf, wf, 1, 3, 3, 0, 0, 0, 2, nullptr, rest, rest_bytes, s, nullptr, nullptr, x8);
}

// =================================================================================================
// Modulated convolution  y = d (.) conv(a (.) x, w)  with one weight tensor shared by every sample (groups = 1, stride 1):
// a [n][cin][t] scales x while it is re-tiled (conv_pack_act_kernel), d [n][cout][to] the accumulators in the epilogue
// (conv_igemm_kernel). The per-sample weights of the reference's grouped formulation (generator_sres.py:44-60) and the
// modulated activation copies (generator_lres.py:117-123) are never formed.
// Backward: dy is re-tiled with the factor d for both gradients; dgrad writes dx' = conv^T(d dy, w) into dx, and one
// streaming pass (modconv_rowdot_kernel) turns it into dx = a dx' while it sums da = sum_hw dx' x. The gradient of d comes
// from sum_hw dy y (= d sum_hw dy conv(a x, w)), a second pass of the same kernel; the caller divides by d.

namespace lvg {
namespace {

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ void from_f32(float& o, float v) { o = v; }
__device__ __forceinline__ void from_f32(__half& o, float v) { o = __float2half_rn(v); }

// r[row] = sum_i u[row][i] * v[row][i] over rows of `len` contiguous elements (fp32 accumulation); scale != nullptr:
// u[row][i] *= scale[row] in place (after it was read). One CTA per row; VEC elements per 16-byte load when rows are aligned.
template <class T, int VEC>
__global__ void __launch_bounds__(256) modconv_rowdot_kernel(T* __restrict__ u, const T* __restrict__ v, const float* __restrict__ scale,
                                                             float* __restrict__ r, int64_t rows, int64_t len)
{
    __shared__ float red[8];
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        T* ur = u + row * len;
        const T* vr = v + row * len;
        const float sc = scale != nullptr ? __ldg(scale + row) : 1.f;
        float acc = 0.f;
        for (int64_t i = (int64_t)threadIdx.x * VEC; i < len; i += 256 * VEC) {
            alignas(16) T ue[VEC], ve[VEC];
            if constexpr (VEC > 1) {
                *reinterpret_cast<uint4*>(ue) = *reinterpret_cast<const uint4*>(ur + i);
                *reinterpret_cast<uint4*>(ve) = __ldg(reinterpret_cast<const uint4*>(vr + i));
            } else {
                ue[0] = ur[i];
                ve[0] = vr[i];
            }
#pragma unroll
            for (int j = 0; j < VEC; j++) {
                const float uf = to_f32(ue[j]);
                acc += uf * to_f32(ve[j]);
                from_f32(ue[j], uf * sc);
            }
            if (scale != nullptr) {
                if constexpr (VEC > 1) *reinterpret_cast<uint4*>(ur + i) = *reinterpret_cast<const uint4*>(ue);
                else ur[i] = ue[0];
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int k = 0; k < 8; k++) s += red[k];
            if (r != nullptr) r[row] = s;
        }
        __syncthreads();
    }
}

int modconv_rowdot(void* u, const void* v, const float* scale, float* r, int dtype, int64_t rows, int64_t len, cudaStream_t s)
{
    int64_t blocks = rows;
    const int64_t cap = (int64_t)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) return LVG_OK;
    const int es = dtype == LVG_F32 ? 4 : 2;
    const bool vec = aligned16(u) && aligned16(v) && (len * es) % 16 == 0;
    if (dtype == LVG_F32) {
        if (vec) modconv_rowdot_kernel<float, 4><<<(unsigned)blocks, 256, 0, s>>>((float*)u, (const float*)v, scale, r, rows, len);
        else modconv_rowdot_kernel<float, 1><<<(unsigned)blocks, 256, 0, s>>>((float*)u, (const float*)v, scale, r, rows, len);
    } else {
        if (vec) modconv_rowdot_kernel<__half, 8><<<(unsigned)blocks, 256, 0, s>>>((__half*)u, (const __half*)v, scale, r, rows, len);
        else modconv_rowdot_kernel<__half, 1><<<(unsigned)blocks, 256, 0, s>>>((__half*)u, (const __half*)v, scale, r, rows, len);
    }
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

// forward and backward run on the engine alone (never the streaming 1x1x1 kernels, which take no factors)
bool modconv_in_envelope(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w)
{
    return cin >= 1 && cout >= 1 && pad_t <= kt - 1 && pad_h <= kh - 1 && pad_w <= kw - 1 &&
           wgrad_in_envelope(dtype, n, 1, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1);
}

inline int64_t round256(int64_t b) { return (b + 255) / 256 * 256; }

}  // namespace
}  // namespace lvg

extern "C" int64_t lvg_modconv_workspace(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h,
                                         int pad_w)
{
    if (!modconv_in_envelope(dtype, n, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w)) return -1;
    const int split = dtype == LVG_F32;
    const int taps = kt * kh * kw;
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    const Geometry gf = geometry(split, n, 1, cin, cout, (int64_t)t * h * wd, taps);          // forward
    const Geometry gd = geometry(split, n, 1, cout, cin, (int64_t)to * ho * wo, taps);        // input gradient
    const WgradPlan q = wgrad_plan(dtype, n, 1, cin, cout, t, h, wd, to, ho, wo, kt, kh, kw);
    const int64_t sep = std::max(std::max(gf.act_bytes + gf.w_bytes, gd.act_bytes + gd.w_bytes), q.a_bytes + q.b_bytes + q.part_bytes);
    const int64_t shared = round256(gd.act_bytes) + std::max(round256(gd.w_bytes) + 256, round256(q.b_bytes) + q.part_bytes + 768);
    return std::max(sep, shared) + 1024;
}

extern "C" int lvg_modconv_fprop(const void* x, const void* w, const float* a, const float* d, void* y, int dtype, int n, int cin, int cout, int t,
                                 int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, void* workspace, int64_t workspace_bytes,
                                 void* stream)
{
    LVG_REQUIRE(x && w && a && y, "modconv_fprop: x, w, a, y must not be NULL");
    if (!modconv_in_envelope(dtype, n, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w)) {
        set_error("modconv_fprop: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    const int taps = kt * kh * kw;
    return run_igemm(x, w, y, dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, (int64_t)cout * cin * taps, (int64_t)cin * taps,
                     taps, 0, nullptr, 0, 0.f, 1.f, -1.f, h, wd, 1, 1, nullptr, workspace, workspace_bytes, (cudaStream_t)stream, a, d);
}

extern "C" int lvg_modconv_backward(const void* x, const void* w, const float* a, const float* d, const void* y, const void* dy, void* dx, void* dw,
                                    float* da, float* dyy, int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                    int pad_t, int pad_h, int pad_w, void* workspace, int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && w && a && dy && dx, "modconv_backward: x, w, a, dy, dx must not be NULL");
    LVG_REQUIRE(!dyy || (y && d), "modconv_backward: sum(dy * y) needs y and d");
    LVG_REQUIRE(workspace && aligned16(workspace), "modconv_backward: workspace must be 16-byte aligned and not NULL");
    if (!modconv_in_envelope(dtype, n, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w)) {
        set_error("modconv_backward: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int split = dtype == LVG_F32 ? 1 : 0;
    const int taps = kt * kh * kw;
    const int to = t + 2 * pad_t - kt + 1, ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    int rc;
    if (dyy) {
        rc = modconv_rowdot(const_cast<void*>(dy), y, nullptr, dyy, dtype, (int64_t)n * cout * to, (int64_t)ho * wo, s);
        if (rc) return rc;
    }
    const Geometry gd = geometry(split, n, 1, cout, cin, (int64_t)to * ho * wo, taps);
    const int64_t w_gs = (int64_t)cout * cin * taps;
    if (wgrad_cpad_a(cout) == round_up(cout, 16)) {
        // one re-tiling of d dy serves both gradients (layout as lvg_convnd_backward: [dy8][dgrad weights | x8, partial sums])
        const int64_t dy8_room = round256(gd.act_bytes);
        const int64_t wp_room = round256(gd.w_bytes) + 256;
        LVG_REQUIRE(workspace_bytes >= dy8_room + wp_room, "modconv_backward: workspace too small");
        unsigned char* dy8 = reinterpret_cast<unsigned char*>(workspace);
        unsigned char* rest = dy8 + dy8_room;
        rc = pack_act(dy, dy8, split, n, cout, gd.cblk, to, ho, wo, ho, wo, 1, s, d);
        if (rc) return rc;
        rc = run_igemm(dy, w, dx, dtype, n, 1, cout, cin, to, ho, wo, kt, kh, kw, kt - 1 - pad_t, kh - 1 - pad_h, kw - 1 - pad_w, w_gs, taps,
                       (int64_t)cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, ho, wo, 1, 1, dy8, rest, wp_room, s);
        if (rc) return rc;
        rc = modconv_rowdot(dx, x, a, da, dtype, (int64_t)n * cin * t, (int64_t)h * wd, s);
        if (rc) return rc;
        return dw ? run_wgrad(x, dy, dw, dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1, dy8, rest, workspace_bytes - dy8_room, s, a)
                  : LVG_OK;
    }
    // output channels that are neither < 128 nor a multiple of 128: the two gradients tile d dy differently, each re-tiles it
    rc = run_igemm(dy, w, dx, dtype, n, 1, cout, cin, to, ho, wo, kt, kh, kw, kt - 1 - pad_t, kh - 1 - pad_h, kw - 1 - pad_w, w_gs, taps,
                   (int64_t)cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, ho, wo, 1, 1, nullptr, workspace, workspace_bytes, s, d);
    if (rc) return rc;
    rc = modconv_rowdot(dx, x, a, da, dtype, (int64_t)n * cin * t, (int64_t)h * wd, s);
    if (rc) return rc;
    return dw ? run_wgrad(x, dy, dw, dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1, nullptr, workspace, workspace_bytes, s, a, d)
              : LVG_OK;
}

// =================================================================================================
// Super-res generator layer  y = d (.) conv(a (.) z, w)  with z = cat(x_prev, cond(lr)) never formed (DESIGN.md 7j): the
// re-tiling pass (conv_pack_cond_kernel) reads x_prev and evaluates the layer's conditioning from the low-res video by its
// plan (sres_cond.cuh: the tap tables and both passes of sres_cond_kernel, in the same order), rounds each value to the
// layer's dtype as lvg_sres_cond does, multiplies it by a and writes X8 as conv_pack_act_kernel does from z: bit for bit
// the modulated convolution of lvg_sres_cond's z. Channel c < C of a sample is x_prev's channel c, channel C + k window + s
// the conditioning of low-res channel k at frame t + s; a block of 8 channels may hold both.
// Backward: dgrad of d dy into all Cin channels (workspace), one streaming pass that dots each row with dtype(x_prev) or
// the conditioning (materialised for its c_lr window channels only, by lvg_sres_cond) for da and writes dx_prev =
// x_dtype(dtype(a dx')) for the x_prev channels, and the weight gradient from X8 rebuilt by the same re-tiling pass.

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
    if (!modconv_in_envelope(dtype, (int)std::min<int64_t>(L.np, 1 << 30), L.cin, cout, 1, L.ah.out, L.aw.out, 1, kh, kw, 0, pad_h, pad_w))
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

// workspace of the forward: [X8][packed weights][statistic partials]
struct SresLayerFwdRooms { int64_t x8, wp, part; };
SresLayerFwdRooms sres_layer_fwd_rooms(const SresLayer& L)
{
    const Geometry g = geometry(L.dtype == LVG_F32, L.np, 1, L.cin, L.cout, L.hw, L.kh * L.kw);
    return {round256(g.act_bytes), round256(g.w_bytes) + 256, round256(sres_layer_pack_ctas(L, g.cblk) * (int64_t)sizeof(double))};
}

// workspace of the backward: [d dy re-tiled (shared by both gradients) | -][dx' over all Cin][conditioning][rest: the
// dgrad weights, then the weight gradient's X8 and partial sums]
struct SresLayerBwdRooms { bool shared; int64_t dy8, dxp, cond, rest, wp; };
SresLayerBwdRooms sres_layer_bwd_rooms(const SresLayer& L)
{
    const int es = L.dtype == LVG_F32 ? 4 : 2;
    const int ho = L.ah.out + 2 * L.pad_h - L.kh + 1, wo = L.aw.out + 2 * L.pad_w - L.kw + 1;
    const Geometry gd = geometry(L.dtype == LVG_F32, L.np, 1, L.cout, L.cin, (int64_t)ho * wo, L.kh * L.kw);
    const WgradPlan q = wgrad_plan(L.dtype, (int)L.np, 1, L.cin, L.cout, 1, L.ah.out, L.aw.out, 1, ho, wo, 1, L.kh, L.kw);
    SresLayerBwdRooms r;
    r.shared = wgrad_cpad_a(L.cout) == round_up(L.cout, 16);
    r.dy8 = r.shared ? round256(gd.act_bytes) : 0;
    r.dxp = round256(L.np * L.cin * L.hw * es);
    r.cond = round256(L.np * (L.cin - L.c) * L.hw * es);
    r.wp = round256(gd.w_bytes) + 256;
    const int64_t wg = (r.shared ? 0 : round256(q.a_bytes)) + round256(q.b_bytes) + q.part_bytes + 768;
    const int64_t dg = r.shared ? r.wp : round256(gd.w_bytes) + gd.act_bytes + 256;
    r.rest = std::max(wg, dg);
    return r;
}

}  // namespace
}  // namespace lvg

extern "C" int64_t lvg_sres_layer_workspace(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                            const int* plan_h, const int* plan_w, int cout, int kh, int kw, int pad_h, int pad_w)
{
    SresLayer L;
    if (!sres_layer_plan(dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h, plan_w, cout, kh, kw, pad_h, pad_w, L)) return -1;
    const SresLayerFwdRooms f = sres_layer_fwd_rooms(L);
    const SresLayerBwdRooms b = sres_layer_bwd_rooms(L);
    return std::max(f.x8 + f.wp + f.part, b.dy8 + b.dxp + b.cond + b.rest) + 1024;
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
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.x8 + r.wp + r.part, "sres_layer_fprop: workspace too small or misaligned");
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
    const int taps = kh * kw;
    return run_igemm(x8, w, y, dtype, (int)L.np, 1, L.cin, cout, 1, L.ah.out, L.aw.out, 1, kh, kw, 0, pad_h, pad_w, (int64_t)cout * L.cin * taps,
                     (int64_t)L.cin * taps, taps, 0, nullptr, 0, 0.f, 1.f, -1.f, L.ah.out, L.aw.out, 1, 1, x8, wp, r.wp, s, nullptr, d);
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
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.dy8 + r.dxp + r.cond + r.rest,
                "sres_layer_backward: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    const int split = dtype == LVG_F32 ? 1 : 0;
    const int taps = kh * kw;
    const int h = L.ah.out, wd = L.aw.out, np = (int)L.np;
    const int ho = h + 2 * pad_h - kh + 1, wo = wd + 2 * pad_w - kw + 1;
    unsigned char* dy8 = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* dxp = dy8 + r.dy8;
    unsigned char* cond = dxp + r.dxp;
    unsigned char* rest = cond + r.cond;
    const int64_t rest_bytes = workspace_bytes - (r.dy8 + r.dxp + r.cond);
    int rc;
    if (dyy) {
        rc = modconv_rowdot(const_cast<void*>(dy), y, nullptr, dyy, dtype, (int64_t)np * cout, (int64_t)ho * wo, s);
        if (rc) return rc;
    }
    // dx' = conv^T(d dy, w) over all Cin channels, as lvg_modconv_backward computes it
    const Geometry gd = geometry(split, np, 1, cout, L.cin, (int64_t)ho * wo, taps);
    const int64_t w_gs = (int64_t)cout * L.cin * taps;
    if (r.shared) {
        rc = pack_act(dy, dy8, split, np, cout, gd.cblk, 1, ho, wo, ho, wo, 1, s, d);
        if (rc) return rc;
        rc = run_igemm(dy, w, dxp, dtype, np, 1, cout, L.cin, 1, ho, wo, 1, kh, kw, 0, kh - 1 - pad_h, kw - 1 - pad_w, w_gs, taps,
                       (int64_t)L.cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, ho, wo, 1, 1, dy8, rest, r.wp, s);
    } else {
        rc = run_igemm(dy, w, dxp, dtype, np, 1, cout, L.cin, 1, ho, wo, 1, kh, kw, 0, kh - 1 - pad_h, kw - 1 - pad_w, w_gs, taps,
                       (int64_t)L.cin * taps, 1, nullptr, 0, 0.f, 1.f, -1.f, ho, wo, 1, 1, nullptr, rest, rest_bytes, s, d);
    }
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
    // dw from X8 of a z rebuilt by the re-tiling pass, in the slot run_wgrad would re-tile x into
    const WgradPlan q = wgrad_plan(dtype, np, 1, L.cin, cout, 1, h, wd, 1, ho, wo, 1, kh, kw);
    unsigned char* x8 = r.shared ? rest : rest + round256(q.a_bytes);
    rc = sres_layer_pack(L, x, x_dtype, lr, lr_strides, f_h, gain_h, f_w, gain_w, a, x8, q.cpad_b / 8, nullptr, s);
    if (rc) return rc;
    return run_wgrad(nullptr, dy, dw, dtype, np, 1, L.cin, cout, 1, h, wd, 1, kh, kw, 0, pad_h, pad_w, 1, r.shared ? dy8 : nullptr, rest,
                     rest_bytes, s, nullptr, r.shared ? nullptr : d, x8);
}
