// Fused filtered leaky ReLU: bias -> up-FIR -> gain*lrelu*clamp (+ 2-bit signs) -> down-FIR in ONE kernel.
//
// The three separable configurations of the super-res generator run the vectorised kernel of filtered_lrelu_v3.cuh
// (semantics and formulation are described there); 1x1 filters without resampling (the ToRGB layer) run an
// element-wise kernel. Filters arrive as device pointers and are staged per CTA in shared memory -- no global
// __constant__ state (the reference's c_fbuf, filtered_lrelu.cu:78), so the op is stream-safe.

#include "common.cuh"
#include "filtered_lrelu_v3.cuh"

namespace lvg {
namespace flv3 {

template <class T, class G, int MODE>
__global__ void __launch_bounds__(kThreads, G::ctas(MODE)) filtered_lrelu_v3_kernel(FlParams p)
{
    extern __shared__ __align__(16) float smem[];
    const Tile t = make_tile<G>(p, blockIdx.x);
    const Smem s = carve<G>(smem);
    const int tid = threadIdx.x;
    stage0<G, MODE>(p, t, s, tid);
    stage1<T, G>(p, t, s, tid);
    __syncthreads();
    stage2<G>(t, s, tid);
    __syncthreads();
    stage3<G, MODE>(p, t, s, tid);
    __syncthreads();
    if (MODE == SIGN_WRITE) stage3_fixup<G>(p, t, tid);
    stage4<G>(t, s, tid);
    __syncthreads();
    stage5<T, G>(p, t, s, tid);
}

template <class T, class G>
static int launch_cfg(FlParams& p, int mode, cudaStream_t s)
{
    fill_launch_constants<G>(p);
    const int64_t tiles = (int64_t)p.tiles_x * p.tiles_y;
    const int64_t blocks = (int64_t)p.n * p.c * tiles;
    // one-multiply block-index decomposition: exact while dividend * divisor < 2^32
    LVG_REQUIRE(blocks <= INT32_MAX && blocks * tiles < (1ll << 32) && (int64_t)p.n * p.c * p.c < (1ll << 32),
                "filtered_lrelu: grid too large");
    const size_t smem = G::smem_bytes(mode);
    void (*k)(FlParams) = nullptr;
    if (mode == SIGN_WRITE)     k = filtered_lrelu_v3_kernel<T, G, SIGN_WRITE>;
    else if (mode == SIGN_READ) k = filtered_lrelu_v3_kernel<T, G, SIGN_READ>;
    else                        k = filtered_lrelu_v3_kernel<T, G, SIGN_NONE>;
    LVG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<(unsigned)blocks, kThreads, smem, s>>>(p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace flv3

namespace {
using namespace flv3;

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

template <class T>
int dispatch(Cfg cfg, FlParams& p, int mode, cudaStream_t s)
{
    switch (cfg) {
        case CFG_1x1:  return launch_1x1<T>(p, mode, s);
        case CFG_U2D2: return launch_cfg<T, Geom<2, 12, 2, 12, 56, 24, 6, 2, 4, 4>>(p, mode, s);
        case CFG_U4D2: return launch_cfg<T, Geom<4, 24, 2, 12, 56, 24, 2, 2, 4, 4>>(p, mode, s);
        case CFG_U2D4: return launch_cfg<T, Geom<2, 12, 4, 24, 31, 16, 8, 6, 4, 2>>(p, mode, s);
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
    if (cfg != CFG_1x1) {
        // the fused kernel computes the leaky ReLU as max(v, v * slope) and stages sign rows with aligned 32-bit loads
        if (!(slope <= 1.f)) {
            set_error("filtered_lrelu: the fused kernel needs slope <= 1 (got %g)", (double)slope);
            return LVG_UNSUPPORTED;
        }
        LVG_REQUIRE(!si || (s_wbytes % 4 == 0 && (reinterpret_cast<uintptr_t>(si) & 3) == 0),
                    "filtered_lrelu: sign rows must be a multiple of 4 bytes and start on a 4-byte boundary");
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
