// Adjoint of conv1's FIR fused with conv0's activation gradient, for a super-res discriminator block (DESIGN.md 7i):
//
//   dz0 = G(h0) (.) FIR^T(dhf),   db0[c] = sum over samples and pixels of dz0[:, c]
//
// dhf: the gradient of the filtered image upfirdn2d(h0, f, padding = 2) ((h + 1) x (w + 1), conv1's input gradient), h0:
// conv0's output (h x w), G: the lrelu / linear slope times gain decided from the sign of h0, zero where the forward clamped
// (bias_act's first-order gradient, bias_act.cu bias_act_elem with G = 1). FIR^T of the correlation with taps g (padding 2)
// is the correlation of dhf with the mirrored taps and padding 1; both axes run as separable passes in shared memory with
// fp32 accumulation, and dz0 is rounded once to the storage type. Replaces upfirdn2d's adjoint (a write and a re-read of
// dh0) and bias_act's gradient pass, and the separate reduction of db0: every CTA sums its tile of the stored dz0 in a
// fixed order into one partial, and a second kernel folds the partials of each channel in a fixed order (no atomics, bitwise
// reproducible).
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "conv_engine.cuh"

namespace lvg {
namespace {

constexpr int kAdjTX = 32, kAdjTY = 8, kAdjPitch = kAdjTX + 4;

template <class T>
__global__ void __launch_bounds__(256) sres_fir_adjoint_act_kernel(const T* __restrict__ dhf, const T* __restrict__ h0, const float* __restrict__ fx,
                                                                    const float* __restrict__ fy, int flip, T* __restrict__ dz, float* __restrict__ part,
                                                                    int h, int w, int lrelu, float alpha, float gain, float clamp)
{
    __shared__ float s_in[kAdjTY + 3][kAdjPitch];
    __shared__ float s_mid[kAdjTY][kAdjPitch];
    __shared__ float s_red[8];
    const int hf = h + 1, wf = w + 1;
    const int j0 = blockIdx.x * kAdjTX, i0 = blockIdx.y * kAdjTY;
    const int64_t plane = blockIdx.z;
    // forward correlation taps g[k] (as conv_pack_fir4_kernel orients them); the adjoint reads them mirrored
    float ax[4], ay[4];
#pragma unroll
    for (int m = 0; m < 4; m++) {
        const int k = 3 - m;
        ax[m] = __ldg(fx + (flip ? k : 3 - k));
        ay[m] = __ldg(fy + (flip ? k : 3 - k));
    }
    const T* src = dhf + plane * hf * wf;
    for (int i = threadIdx.x; i < (kAdjTY + 3) * (kAdjTX + 3); i += 256) {
        const int col = i % (kAdjTX + 3), r = i / (kAdjTX + 3);
        const int y = i0 - 1 + r, x = j0 - 1 + col;
        s_in[r][col] = (y >= 0 && y < hf && x >= 0 && x < wf) ? (float)src[(int64_t)y * wf + x] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kAdjTY * (kAdjTX + 3); i += 256) {
        const int col = i % (kAdjTX + 3), r = i / (kAdjTX + 3);
        float v = 0.f;
#pragma unroll
        for (int m = 0; m < 4; m++) v = fmaf(ay[m], s_in[r + m][col], v);
        s_mid[r][col] = v;
    }
    __syncthreads();
    const int tx = threadIdx.x % kAdjTX, ty = threadIdx.x / kAdjTX;
    const int i = i0 + ty, j = j0 + tx;
    float stored = 0.f;
    if (i < h && j < w) {
        float v = 0.f;
#pragma unroll
        for (int m = 0; m < 4; m++) v = fmaf(ax[m], s_mid[ty][tx + m], v);
        const int64_t off = plane * h * w + (int64_t)i * w + j;
        const float y = (float)h0[off];
        // bias_act_elem, G = 1: (y > 0 ? v : v * alpha) * gain, zero where the forward clamped
        float o = (lrelu && !(y > 0.f)) ? v * alpha : v;
        o *= gain;
        if (clamp >= 0.f && !(y > -clamp && y < clamp)) o = 0.f;
        const T t = (T)o;
        dz[off] = t;
        stored = (float)t;
    }
    // fixed-order tile sum: a shuffle tree per warp, then the 8 warps in order
#pragma unroll
    for (int d = 16; d > 0; d /= 2) stored += __shfl_down_sync(0xffffffffu, stored, d);
    if (threadIdx.x % 32 == 0) s_red[threadIdx.x / 32] = stored;
    __syncthreads();
    if (threadIdx.x == 0) {
        float acc = 0.f;
        for (int k = 0; k < 8; k++) acc += s_red[k];
        part[plane * (gridDim.x * gridDim.y) + blockIdx.y * gridDim.x + blockIdx.x] = acc;
    }
}

// db[c] = sum over samples n, then tiles t, of part[(n c_total + c) tiles + t], in that order
__global__ void __launch_bounds__(128) sres_fir_adjoint_fold_kernel(const float* __restrict__ part, float* __restrict__ db, int n, int c, int tiles)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= c) return;
    float acc = 0.f;
    for (int s = 0; s < n; s++) {
        const float* p = part + ((int64_t)s * c + ch) * tiles;
        for (int t = 0; t < tiles; t++) acc += p[t];
    }
    db[ch] = acc;
}

int64_t adj_tiles(int h, int w) { return (int64_t)((w + kAdjTX - 1) / kAdjTX) * ((h + kAdjTY - 1) / kAdjTY); }

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

// conv1: the stride-2 3x3 convolution of the filtered (h + 1) x (wd + 1) image
ConvShape conv1_shape(int dtype, int n, int cin, int cout, int h, int wd) { return {dtype, n, 1, cin, cout, 1, h + 1, wd + 1, 1, 3, 3, 0, 0, 0, 2}; }

// workspace of conv1's backward: [X8 of the filtered image][the larger of the input gradient's and the weight gradient's]
struct Conv1BwdRooms {
    int64_t x8, rest;
    int64_t total() const { return x8 + rest; }
};
Conv1BwdRooms conv1_bwd_rooms(const ConvShape& sh)
{
    const WgradPlan q = wgrad_plan(sh);
    return {round256(q.b_bytes), std::max(igemm_rooms(dgrad_job(sh, nullptr, nullptr, nullptr)).total(), wgrad_rooms(q, false).total())};
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_sres_dblock_fir_adjoint_act_workspace(int dtype, int n, int c, int h, int w)
{
    if ((dtype != LVG_F16 && dtype != LVG_F32) || n < 1 || c < 1 || h < 1 || w < 1 || (int64_t)n * c > 65535) return -1;
    return (int64_t)n * c * adj_tiles(h, w) * 4 + 256;
}

extern "C" int lvg_sres_dblock_fir_adjoint_act(const void* dhf, const void* h0, const float* fx, const float* fy, int flip, void* dz, float* db,
                                               void* workspace, int64_t workspace_bytes, int dtype, int n, int c, int h, int w, int act, float alpha,
                                               float gain, float clamp, void* stream)
{
    LVG_REQUIRE(dhf && h0 && fx && fy && dz, "sres_dblock_fir_adjoint_act: dhf, h0, fx, fy, dz must not be NULL");
    const int64_t need = lvg_sres_dblock_fir_adjoint_act_workspace(dtype, n, c, h, w);
    if (need < 0 || (act != 1 && act != 2)) {
        set_error("sres_dblock_fir_adjoint_act: outside the kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(workspace && workspace_bytes >= need, "sres_dblock_fir_adjoint_act: workspace too small");
    cudaStream_t s = (cudaStream_t)stream;
    float* sink = reinterpret_cast<float*>(workspace);          // the per-CTA partials of db (written whether or not db is wanted)
    const dim3 grid((unsigned)((w + kAdjTX - 1) / kAdjTX), (unsigned)((h + kAdjTY - 1) / kAdjTY), (unsigned)(n * c));
    if (dtype == LVG_F32)
        sres_fir_adjoint_act_kernel<float><<<grid, 256, 0, s>>>((const float*)dhf, (const float*)h0, fx, fy, flip, (float*)dz, sink, h, w, act == 2,
                                                                  alpha, gain, clamp);
    else
        sres_fir_adjoint_act_kernel<__half><<<grid, 256, 0, s>>>((const __half*)dhf, (const __half*)h0, fx, fy, flip, (__half*)dz, sink, h, w, act == 2,
                                                                   alpha, gain, clamp);
    LVG_LAUNCH_CHECK();
    if (db) {
        sres_fir_adjoint_fold_kernel<<<(c + 127) / 128, 128, 0, s>>>(sink, db, n, c, (int)adj_tiles(h, w));
        LVG_LAUNCH_CHECK();
    }
    return LVG_OK;
}

// ---- conv1 of a super-res discriminator block (conv2d_resample with down = 2, a 3x3 kernel and padding 1): the 4-tap FIR
// with padding 2 runs inside the re-tiling pass (conv_pack_fir4_kernel), the stride-2 convolution and its bias_act epilogue
// on the engine as lvg_convnd_fprop runs them. Workspace: the rooms of that job, with X8 of the filtered image in its slot.
extern "C" int64_t lvg_sres_dblock_conv1_workspace(int dtype, int n, int cin, int cout, int h, int wd)
{
    if ((dtype != LVG_F16 && dtype != LVG_F32) || n < 1 || cin < 1 || cout < 1 || h < 2 || wd < 2) return -1;
    const int hf = h + 1, wf = wd + 1;
    const Geometry g = geometry(dtype == LVG_F32, n, 1, cin, cout, (int64_t)hf * wf, 9);
    if ((int64_t)n * g.cblk > 65535 || (int64_t)n * g.nblk >= (1ll << 31) || wf - 2 > 4 * (128 - 2)) return -1;
    return igemm_rooms(fprop_job(conv1_shape(dtype, n, cin, cout, h, wd), nullptr, nullptr, nullptr)).total();
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
    IgemmJob j = fprop_job(conv1_shape(dtype, n, cin, cout, h, wd), nullptr, w, y);
    unsigned char* x8 = reinterpret_cast<unsigned char*>(workspace) + igemm_rooms(j).wp;
    {
        const dim3 grid((unsigned)((wf + kFirTX - 1) / kFirTX), (unsigned)((hf + kFirTY - 1) / kFirTY), (unsigned)(n * g.cblk));
        if (split) conv_pack_fir4_kernel<float, true><<<grid, 256, 0, s>>>((const float*)x, (uint4*)x8, cin, g.cblk, h, wd, fx, fy, flip);
        else conv_pack_fir4_kernel<__half, false><<<grid, 256, 0, s>>>((const __half*)x, (uint4*)x8, cin, g.cblk, h, wd, fx, fy, flip);
        LVG_LAUNCH_CHECK();
    }
    j.x8_pre = x8;
    j.bias = bias; j.act = act; j.alpha = alpha; j.gain = gain; j.clamp = clamp;
    return run_igemm(j, workspace, workspace_bytes, s);
}

// ---- conv1's backward: dhf = the input gradient of the strided convolution (the filtered image's gradient, (h + 1) x (wd + 1),
// lvg_convnd_dgrad), and dw from the weight-gradient kernel with its B operand re-tiled straight from x by
// conv_pack_fir4_kernel (the filtered image is recomputed into X8, never into NCHW).
extern "C" int64_t lvg_sres_dblock_conv1_backward_workspace(int dtype, int n, int cin, int cout, int h, int wd)
{
    if (lvg_sres_dblock_conv1_workspace(dtype, n, cin, cout, h, wd) < 0) return -1;
    const ConvShape sh = conv1_shape(dtype, n, cin, cout, h, wd);
    if (!sh.wgrad_ok()) return -1;
    return conv1_bwd_rooms(sh).total();
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
    const ConvShape sh = conv1_shape(dtype, n, cin, cout, h, wd);
    const Conv1BwdRooms r = conv1_bwd_rooms(sh);
    unsigned char* x8 = reinterpret_cast<unsigned char*>(workspace);
    unsigned char* rest = x8 + r.x8;
    const int64_t rest_bytes = workspace_bytes - r.x8;
    if (dhf) {
        const int rc = lvg_convnd_dgrad(dy, w, dhf, dtype, n, 1, cin, cout, 1, hf, wf, 1, 3, 3, 0, 0, 0, 2, rest, rest_bytes, stream);
        if (rc) return rc;
    }
    if (!dw) return LVG_OK;
    const WgradPlan q = wgrad_plan(sh);
    const int cblk = q.cpad_b / 8;
    LVG_REQUIRE((int64_t)n * cblk <= 65535, "sres_dblock_conv1_backward: too many channel blocks");
    {
        const dim3 grid((unsigned)((wf + kFirTX - 1) / kFirTX), (unsigned)((hf + kFirTY - 1) / kFirTY), (unsigned)(n * cblk));
        if (q.split) conv_pack_fir4_kernel<float, true><<<grid, 256, 0, s>>>((const float*)x, (uint4*)x8, cin, cblk, h, wd, fx, fy, flip);
        else conv_pack_fir4_kernel<__half, false><<<grid, 256, 0, s>>>((const __half*)x, (uint4*)x8, cin, cblk, h, wd, fx, fy, flip);
        LVG_LAUNCH_CHECK();
    }
    return run_wgrad(sh, nullptr, dy, dw, WgradInputs{nullptr, x8, nullptr, nullptr}, rest, rest_bytes, s);
}
