// Modulated convolution  y = d (.) conv(a (.) x, w)  with one weight tensor shared by every sample (groups = 1, stride 1):
// a [n][cin][t] scales x while it is re-tiled (conv_pack_act_kernel), d [n][cout][to] the accumulators in the epilogue
// (conv_igemm_kernel). The per-sample weights of the reference's grouped formulation (generator_sres.py:44-60) and the
// modulated activation copies (generator_lres.py:117-123) are never formed.
// Backward: dy is re-tiled with the factor d for both gradients; dgrad writes dx' = conv^T(d dy, w) into dx, and one
// streaming pass (modconv_rowdot_kernel) turns it into dx = a dx' while it sums da = sum_hw dx' x. The gradient of d comes
// from sum_hw dy y (= d sum_hw dy conv(a x, w)), a second pass of the same kernel; the caller divides by d.
#include <algorithm>

#include "common.cuh"
#include "conv_engine.cuh"

namespace lvg {
namespace {

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

}  // namespace

// forward and backward run on the engine alone (never the streaming 1x1x1 kernels, which take no factors)
bool modconv_in_envelope(const ConvShape& s) { return s.cin >= 1 && s.cout >= 1 && s.dgrad_ok() && s.wgrad_ok(); }

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

}  // namespace lvg

using namespace lvg;

// sizes lvg_modconv_fprop and lvg_modconv_backward
extern "C" int64_t lvg_modconv_workspace(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h,
                                         int pad_w)
{
    const ConvShape sh = {dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!modconv_in_envelope(sh)) return -1;
    return std::max(igemm_rooms(fprop_job(sh, nullptr, nullptr, nullptr)).total(), backward_workspace(sh));
}

extern "C" int lvg_modconv_fprop(const void* x, const void* w, const float* a, const float* d, void* y, int dtype, int n, int cin, int cout, int t,
                                 int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, void* workspace, int64_t workspace_bytes,
                                 void* stream)
{
    LVG_REQUIRE(x && w && a && y, "modconv_fprop: x, w, a, y must not be NULL");
    const ConvShape sh = {dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!modconv_in_envelope(sh)) {
        set_error("modconv_fprop: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    IgemmJob j = fprop_job(sh, x, w, y);
    j.in_scale = a; j.out_scale = d;
    return run_igemm(j, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int lvg_modconv_backward(const void* x, const void* w, const float* a, const float* d, const void* y, const void* dy, void* dx, void* dw,
                                    float* da, float* dyy, int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                    int pad_t, int pad_h, int pad_w, void* workspace, int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && w && a && dy && dx, "modconv_backward: x, w, a, dy, dx must not be NULL");
    LVG_REQUIRE(!dyy || (y && d), "modconv_backward: sum(dy * y) needs y and d");
    LVG_REQUIRE(workspace && aligned16(workspace), "modconv_backward: workspace must be 16-byte aligned and not NULL");
    const ConvShape sh = {dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
    if (!modconv_in_envelope(sh)) {
        set_error("modconv_backward: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    if (dyy) {
        rc = modconv_rowdot(const_cast<void*>(dy), y, nullptr, dyy, dtype, (int64_t)n * cout * sh.to(), (int64_t)sh.ho() * sh.wo(), s);
        if (rc) return rc;
    }
    Backward b;
    rc = backward_dgrad(sh, dy, d, w, dx, workspace, workspace_bytes, s, b);
    if (rc) return rc;
    rc = modconv_rowdot(dx, x, a, da, dtype, (int64_t)n * cin * t, (int64_t)h * wd, s);
    if (rc) return rc;
    return dw ? backward_wgrad(sh, b, x, dy, d, dw, a, nullptr, s) : LVG_OK;
}
