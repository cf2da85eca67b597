// Grouped 2-D convolution entry points (fp16, stride 1, 3x3 or 1x1) of the conv2d plugin, run on the implicit-GEMM engine
// of conv_igemm.cu: a 2-D convolution is its T = kt = 1 case, with the same NCHW / [G*Cout][Cin][kh][kw] memory layout.

#include "common.cuh"

namespace lvg {
namespace {

bool supported(int dtype, int kh, int kw, int stride)
{
    return dtype == LVG_F16 && stride == 1 && ((kh == 3 && kw == 3) || (kh == 1 && kw == 1));
}

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_conv2d_fprop_workspace(int dtype, int n, int groups, int cin, int cout, int h, int wd, int kh, int kw,
                                              int stride, int pad_h, int pad_w)
{
    if (!supported(dtype, kh, kw, stride) || n < 1) return -1;
    // enough for either direction
    return lvg_convnd_workspace(dtype, n, groups, cin, cout, 1, h, wd, 1, kh, kw, 0, pad_h, pad_w);
}

extern "C" int lvg_conv2d_fprop(const void* x, const void* w, void* y, int dtype, int n, int groups, int cin, int cout,
                                int h, int wd, int kh, int kw, int stride, int pad_h, int pad_w, void* workspace,
                                int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(x && w && y, "conv2d_fprop: x, w, y must not be NULL");
    if (!supported(dtype, kh, kw, stride) || n < 1 || pad_h < 0 || pad_w < 0) {
        set_error("conv2d_fprop: outside the tensor-core kernel's envelope (fp16, stride 1, 3x3 or 1x1)");
        return LVG_UNSUPPORTED;
    }
    return lvg_convnd_fprop(x, w, y, dtype, n, groups, cin, cout, 1, h, wd, 1, kh, kw, 0, pad_h, pad_w, 1, nullptr, 0, 0.f, 1.f, -1.f,
                            workspace, workspace_bytes, stream);
}

extern "C" int lvg_conv2d_dgrad(const void* dy, const void* w, void* dx, int dtype, int n, int groups, int cin, int cout,
                                int h, int wd, int kh, int kw, int stride, int pad_h, int pad_w, void* workspace,
                                int64_t workspace_bytes, void* stream)
{
    LVG_REQUIRE(dy && w && dx, "conv2d_dgrad: dy, w, dx must not be NULL");
    if (!supported(dtype, kh, kw, stride) || n < 1 || pad_h > kh - 1 || pad_w > kw - 1 || pad_h < 0 || pad_w < 0) {
        set_error("conv2d_dgrad: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    return lvg_convnd_dgrad(dy, w, dx, dtype, n, groups, cin, cout, 1, h, wd, 1, kh, kw, 0, pad_h, pad_w, 1, workspace, workspace_bytes,
                            stream);
}

// The weight gradient takes no workspace argument: the engine's re-tiled operands and partial sums live in a
// stream-ordered allocation for the duration of the call.
extern "C" int lvg_conv2d_wgrad(const void* x, const void* dy, void* dw, int dtype, int n, int groups, int cin, int cout,
                                int h, int wd, int kh, int kw, int stride, int pad_h, int pad_w, void* stream)
{
    LVG_REQUIRE(x && dy && dw, "conv2d_wgrad: x, dy, dw must not be NULL");
    if (!supported(dtype, kh, kw, stride) || n < 1 || pad_h < 0 || pad_w < 0) {
        set_error("conv2d_wgrad: outside the tensor-core kernel's envelope (fp16, stride 1, 3x3 or 1x1)");
        return LVG_UNSUPPORTED;
    }
    const int64_t need = lvg_convnd_wgrad_workspace(dtype, n, groups, cin, cout, 1, h, wd, 1, kh, kw, 0, pad_h, pad_w);
    if (need < 0) {
        set_error("conv2d_wgrad: outside the tensor-core kernel's envelope");
        return LVG_UNSUPPORTED;
    }
    cudaStream_t s = (cudaStream_t)stream;
    void* ws = nullptr;
    LVG_CUDA(cudaMallocAsync(&ws, (size_t)need, s));
    const int rc = lvg_convnd_wgrad(x, dy, dw, dtype, n, groups, cin, cout, 1, h, wd, 1, kh, kw, 0, pad_h, pad_w, 1, ws, need, stream);
    LVG_CUDA(cudaFreeAsync(ws, s));
    return rc;
}
