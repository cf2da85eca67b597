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

#include "common.cuh"

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
