// Pointwise (1x1x1) convolutions with few channels, fp32, as streaming SIMT kernels.
//
// The low-res networks hold a dozen 1x1x1 convolutions with 3..128 channels over 3-4 million pixels (to/from RGB layers,
// skip connections: generator_lres.py:544-592, discriminator_lres.py:135-213). They are HBM-bound by a wide margin
// (<= 8192 multiply-adds per pixel against 8 bytes per channel and pixel), and the tensor-core engine is the wrong tool for
// them: it re-tiles the input into bf16 hi/lo channel blocks first (one extra read + write of the tensor), pads the
// 3..64 output channels to a 128-row MMA and runs three products per term (tools/lres_conv_table.py compares the two per
// layer). These kernels read x once, write y once, and multiply in exact fp32:
//   forward         y[n][co][p] = sum_ci W[co][ci] * x[n][ci][p]
//   input gradient  the same kernel on dy with the transposed weight view
// The weight gradient of these layers runs on the engine.
// Envelope: 1x1x1, stride 1, no padding, groups 1, fp32, cin * cout <= 4096, pixels per sample a multiple of 4,
// 16-byte aligned tensors; every other 1x1x1 forward / input gradient runs on the pointwise wgmma kernels (conv_pw_tc.cu),
// everything else on the engine (lvg_convnd_route in conv_igemm.cu checks pw_supported first).
#include "common.cuh"

namespace lvg {
namespace {

constexpr int kPwThreads = 256;
constexpr int kPwCiChunk = 64;          // input channels staged per pass

__device__ __forceinline__ float2 pw_fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// CO_T output channels per thread (even), CT channel threads; a CTA covers PXT = (256 / CT) * 4 pixels of one sample.
// ws: weights [ci][COP] (COP = CO_T * CT, zero padded), xs: [ci chunk][PXT].
template <int CO_T, int CT>
__global__ void __launch_bounds__(kPwThreads, 2) pw_conv_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y,
                                                                int cin, int cout, int64_t P, int tiles, int64_t w_sco, int64_t w_sci)
{
    constexpr int PT = kPwThreads / CT, PXT = PT * 4, COP = CO_T * CT;
    extern __shared__ __align__(16) float smem[];
    float* ws = smem;                               // [cin][COP]
    float* xs = smem + (size_t)cin * COP;           // [kPwCiChunk][PXT]
    const int n = blockIdx.x / tiles, tile = blockIdx.x - n * tiles;
    const int64_t p0 = (int64_t)tile * PXT;
    const int pt = threadIdx.x % PT, cg = threadIdx.x / PT;
    for (int i = threadIdx.x; i < cin * COP; i += kPwThreads) {
        const int ci = i / COP, co = i - ci * COP;
        ws[i] = co < cout ? w[co * w_sco + ci * w_sci] : 0.f;
    }
    float2 acc[CO_T / 2][4];
#pragma unroll
    for (int j = 0; j < CO_T / 2; j++)
#pragma unroll
        for (int k = 0; k < 4; k++) acc[j][k] = make_float2(0.f, 0.f);
    const float* xn = x + (int64_t)n * cin * P;
    for (int c0 = 0; c0 < cin; c0 += kPwCiChunk) {
        const int cn = min(kPwCiChunk, cin - c0);
        __syncthreads();                            // previous chunk consumed (and, first time, nothing)
        for (int i = threadIdx.x; i < cn * PT; i += kPwThreads) {
            const int ci = i / PT, q = i - ci * PT;
            const int64_t p = p0 + 4 * q;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < P) v = *reinterpret_cast<const float4*>(xn + (int64_t)(c0 + ci) * P + p);
            *reinterpret_cast<float4*>(xs + ci * PXT + 4 * q) = v;
        }
        __syncthreads();
        const float* wrow = ws + (size_t)c0 * COP + cg * CO_T;
#pragma unroll 4
        for (int ci = 0; ci < cn; ci++) {
            const float4 xv = *reinterpret_cast<const float4*>(xs + ci * PXT + 4 * pt);
            const float2 x0 = make_float2(xv.x, xv.x), x1 = make_float2(xv.y, xv.y), x2 = make_float2(xv.z, xv.z), x3 = make_float2(xv.w, xv.w);
#pragma unroll
            for (int j = 0; j < CO_T / 2; j++) {
                const float2 wp = *reinterpret_cast<const float2*>(wrow + ci * COP + 2 * j);
                acc[j][0] = pw_fma2(wp, x0, acc[j][0]);
                acc[j][1] = pw_fma2(wp, x1, acc[j][1]);
                acc[j][2] = pw_fma2(wp, x2, acc[j][2]);
                acc[j][3] = pw_fma2(wp, x3, acc[j][3]);
            }
        }
    }
    const int64_t p = p0 + 4 * pt;
    if (p < P) {
        float* yn = y + (int64_t)n * cout * P + p;
#pragma unroll
        for (int j = 0; j < CO_T / 2; j++) {
            const int co = cg * CO_T + 2 * j;
            if (co < cout) *reinterpret_cast<float4*>(yn + (int64_t)co * P) = make_float4(acc[j][0].x, acc[j][1].x, acc[j][2].x, acc[j][3].x);
            if (co + 1 < cout) *reinterpret_cast<float4*>(yn + (int64_t)(co + 1) * P) = make_float4(acc[j][0].y, acc[j][1].y, acc[j][2].y, acc[j][3].y);
        }
    }
}

template <int CO_T, int CT>
int pw_launch(const float* x, const float* w, float* y, int n, int cin, int cout, int64_t P, int64_t w_sco, int64_t w_sci, cudaStream_t s)
{
    constexpr int PXT = (kPwThreads / CT) * 4, COP = CO_T * CT;
    const int tiles = (int)((P + PXT - 1) / PXT);
    const size_t smem = ((size_t)cin * COP + (size_t)kPwCiChunk * PXT) * sizeof(float);
    LVG_REQUIRE((int64_t)n * tiles <= INT32_MAX && smem <= 112 * 1024, "pointwise conv: launch out of range");
    LVG_CUDA(cudaFuncSetAttribute(pw_conv_kernel<CO_T, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    pw_conv_kernel<CO_T, CT><<<(unsigned)(n * tiles), kPwThreads, smem, s>>>(x, w, y, cin, cout, P, tiles, w_sco, w_sci);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace

// LVG_POINTWISE=0 keeps every convolution on the tensor-core engine (A/B measurements)
bool pw_enabled()
{
    static int v = -1;
    if (v < 0) { const char* e = getenv("LVG_POINTWISE"); v = (e && e[0] == '0') ? 0 : 1; }
    return v == 1;
}

// Channel limits: forward / input gradient take these kernels up to cin * cout = 4096, where the engine's re-tiling and
// padding cost more than the layer's traffic. The limits have not been re-measured on the H100 (tools/lres_conv_table.py
// compares both paths).
bool pw_supported(int dtype, int groups, int cin, int cout, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, int64_t P)
{
    return pw_enabled() && dtype == LVG_F32 && groups == 1 && kt == 1 && kh == 1 && kw == 1 && pad_t == 0 && pad_h == 0 && pad_w == 0 && stride == 1 &&
           cin >= 1 && cout >= 1 && cin <= 128 && cout <= 128 && cin * cout <= 4096 && P % 4 == 0 && P >= 4;
}

// y[n][co][p] = sum_ci w[co * w_sco + ci * w_sci] * x[n][ci][p]   (forward: w_sco = cin, w_sci = 1; input gradient: swapped roles)
int pw_conv(const float* x, const float* w, float* y, int n, int cin, int cout, int64_t P, int64_t w_sco, int64_t w_sci, cudaStream_t s)
{
    LVG_REQUIRE(aligned16(x) && aligned16(y), "pointwise conv: tensors must be 16-byte aligned");
    if (cout <= 8)  return pw_launch<2, 4>(x, w, y, n, cin, cout, P, w_sco, w_sci, s);
    if (cout <= 32) return pw_launch<8, 4>(x, w, y, n, cin, cout, P, w_sco, w_sci, s);
    if (cout <= 64) return pw_launch<16, 4>(x, w, y, n, cin, cout, P, w_sco, w_sci, s);
    return pw_launch<16, 8>(x, w, y, n, cin, cout, P, w_sco, w_sci, s);
}

}  // namespace lvg
