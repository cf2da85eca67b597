// First modulated convolution of the low-res generator's residual block with its bias_act and the next layer's magnitude
// statistic (generator_lres.py:568-575):
//   y = clamp(act(d (.) conv(a (.) x, w) + b) * gain)
// on the convolution engine: a scales x while it is re-tiled, d, the bias, the activation, the gain and the clamp are applied
// to the accumulators in the epilogue (conv_igemm_kernel's out_scale instances), so the pre-activation is never stored.
// On request one more pass reads y back and sums its squares (conv0_sumsq_kernel: per-CTA partials over a fixed grid, then
// conv0_fold_kernel in a fixed order): sum y^2 as stored, the statistic input_magnitude_ema_1 takes from y. (Summing in the
// engine's epilogue instead raised the register count of every out_scale instance of conv_igemm_kernel; the engine is
// left as it is.)
// Backward (first order), with dz = G(y) dy the gradient of the pre-activation (bias_act's rule, from y):
//   conv0_rows_kernel  one pass over (dy, y) per (n, c, t) row: s1 = sum G(y) dy, s2 = sum G(y) dy (z(y) - b) with z(y) the
//                      pre-activation recovered from y (where y is not clamped; G = 0 elsewhere); dd = s2 / d
//   conv0_db_kernel    db[c] = sum_{n,t} s1 in a fixed order
//   backward_dgrad     dy re-tiled as dy G(y) d (dz is never written), dx' = conv^T(dz d, w)
//   modconv_rowdot     dx = a dx', da = sum_hw dx' x
//   backward_wgrad     dw from the same tiles (or dy re-tiled again with the same gate)
#include <algorithm>

#include "common.cuh"
#include "conv_engine.cuh"

namespace lvg {
namespace {

constexpr int kSumsqCtasPerSm = 4;

// part[blockIdx.x] = sum of y[i]^2 over the CTA's grid-stride share of y (fixed order for a fixed grid)
template <class T, int VEC>
__global__ void __launch_bounds__(256) conv0_sumsq_kernel(const T* __restrict__ y, int64_t n, float* __restrict__ part)
{
    __shared__ float red[8];
    float s = 0.f;
    const int64_t nv = n / VEC;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < nv; i += (int64_t)gridDim.x * 256) {
        alignas(16) T v[VEC];
        if constexpr (VEC > 1) *reinterpret_cast<uint4*>(v) = __ldg(reinterpret_cast<const uint4*>(y) + i);
        else v[0] = y[i];
#pragma unroll
        for (int j = 0; j < VEC; j++) s += to_f32(v[j]) * to_f32(v[j]);
    }
    if (blockIdx.x == 0)                                        // the tail that does not fill a vector
        for (int64_t i = nv * VEC + threadIdx.x; i < n; i += 256) s += to_f32(y[i]) * to_f32(y[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int k = 0; k < 8; k++) t += red[k];
        part[blockIdx.x] = t;
    }
}

// sumsq[0] = sum of part[0, n) in a fixed order (one CTA; fp64 accumulation)
__global__ void __launch_bounds__(256) conv0_fold_kernel(const float* __restrict__ part, int64_t n, float* __restrict__ sumsq)
{
    __shared__ double red[256];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += 256) s += (double)part[i];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) sumsq[0] = (float)red[0];
}

struct RowArgs {
    int act;
    float alpha, gain, inv_gain, clamp;
};

// one CTA per row (n, c, t) of len = ho * wo elements: s1[row] = sum G(y) dy, dd[row] = (sum G(y) dy (z(y) - b[c])) / d[row]
template <class T, int VEC>
__global__ void __launch_bounds__(256) conv0_rows_kernel(const T* __restrict__ dy, const T* __restrict__ y, const float* __restrict__ b,
                                                         const float* __restrict__ d, float* __restrict__ s1, float* __restrict__ dd, int64_t rows,
                                                         int64_t len, int cout, int to, RowArgs ra)
{
    __shared__ float red[2][8];
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        const T* dyr = dy + row * len;
        const T* yr = y + row * len;
        const float bc = b != nullptr ? __ldg(b + (row / to) % cout) : 0.f;
        float a1 = 0.f, a2 = 0.f;
        for (int64_t i = (int64_t)threadIdx.x * VEC; i < len; i += 256 * VEC) {
            alignas(16) T ge[VEC], ye[VEC];
            if constexpr (VEC > 1) {
                *reinterpret_cast<uint4*>(ge) = __ldg(reinterpret_cast<const uint4*>(dyr + i));
                *reinterpret_cast<uint4*>(ye) = __ldg(reinterpret_cast<const uint4*>(yr + i));
            } else {
                ge[0] = dyr[i];
                ye[0] = yr[i];
            }
#pragma unroll
            for (int j = 0; j < VEC; j++) {
                const float yv = to_f32(ye[j]);
                const float r = yv * ra.inv_gain;                       // the activation's output before the gain
                const bool neg = ra.act == 2 && !(r > 0.f);
                float g = neg ? to_f32(ge[j]) * ra.alpha : to_f32(ge[j]);
                g *= ra.gain;
                if (ra.clamp >= 0.f && !(yv > -ra.clamp && yv < ra.clamp)) g = 0.f;
                if (g != 0.f) {
                    a1 += g;
                    a2 += g * ((neg ? r / ra.alpha : r) - bc);          // z(y) - b: the modulated convolution's output
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a1 += __shfl_xor_sync(0xffffffffu, a1, o);
            a2 += __shfl_xor_sync(0xffffffffu, a2, o);
        }
        if (threadIdx.x % 32 == 0) { red[0][threadIdx.x / 32] = a1; red[1][threadIdx.x / 32] = a2; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float t1 = 0.f, t2 = 0.f;
            for (int k = 0; k < 8; k++) { t1 += red[0][k]; t2 += red[1][k]; }
            s1[row] = t1;
            if (dd != nullptr) dd[row] = t2 / __ldg(d + row);
        }
        __syncthreads();
    }
}

// db[c] = sum over n, then t of s1[n][c][t] (fixed order)
__global__ void __launch_bounds__(256) conv0_db_kernel(const float* __restrict__ s1, float* __restrict__ db, int n, int cout, int to)
{
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= cout) return;
    float s = 0.f;
    for (int i = 0; i < n; i++)
        for (int t = 0; t < to; t++) s += s1[((int64_t)i * cout + c) * to + t];
    db[c] = s;
}

ConvShape conv0_shape(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w)
{
    return {dtype, n, 1, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, 1};
}

// the op's envelope: the modulated convolution's, an output of the input's frame count and linear / lrelu
bool conv0_ok(const ConvShape& s, int act) { return modconv_in_envelope(s) && s.to() == s.t && (act == 1 || act == 2); }

// workspace of the forward: [the engine's job][per-CTA partial sums of squares]
struct FpropRooms {
    int64_t job, part;
    int64_t total() const { return job + part; }
};
FpropRooms fprop_rooms(const ConvShape& s, int sms)
{
    return {round256(igemm_rooms(fprop_job(s, nullptr, nullptr, nullptr)).total()), round256((int64_t)sms * kSumsqCtasPerSm * (int64_t)sizeof(float))};
}
// (the size query does not touch the device: it reserves partials for up to 256 SMs)
constexpr int kMaxSms = 256;

// sumsq[0] = sum of y^2 over n elements: partials, then the fold
int sumsq_of(const void* y, int dtype, int64_t n, float* part, float* sumsq, cudaStream_t s)
{
    const int ctas = num_sms() * kSumsqCtasPerSm;
    const bool vec = aligned16(y);
    if (dtype == LVG_F32) {
        if (vec) conv0_sumsq_kernel<float, 4><<<ctas, 256, 0, s>>>((const float*)y, n, part);
        else conv0_sumsq_kernel<float, 1><<<ctas, 256, 0, s>>>((const float*)y, n, part);
    } else {
        if (vec) conv0_sumsq_kernel<__half, 8><<<ctas, 256, 0, s>>>((const __half*)y, n, part);
        else conv0_sumsq_kernel<__half, 1><<<ctas, 256, 0, s>>>((const __half*)y, n, part);
    }
    LVG_LAUNCH_CHECK();
    conv0_fold_kernel<<<1, 256, 0, s>>>(part, ctas, sumsq);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

// workspace of the backward: [s1 per row][the engine's backward]
int64_t rows_room(const ConvShape& s) { return round256((int64_t)s.n * s.cout * s.to() * (int64_t)sizeof(float)); }

}  // namespace
}  // namespace lvg

using namespace lvg;

extern "C" int64_t lvg_gblock_conv0_workspace(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h,
                                              int pad_w)
{
    const ConvShape sh = conv0_shape(dtype, n, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w);
    if (!conv0_ok(sh, 2)) return -1;
    return std::max(fprop_rooms(sh, kMaxSms).total(), rows_room(sh) + backward_workspace(sh));
}

extern "C" int lvg_gblock_conv0_fprop(const void* x, const void* w, const float* a, const float* d, const float* b, void* y, float* sumsq, int dtype,
                                      int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int act,
                                      float alpha, float gain, float clamp, void* workspace, int64_t workspace_bytes, void* stream)
{
    const ConvShape sh = conv0_shape(dtype, n, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w);
    if (!conv0_ok(sh, act)) {
        set_error("gblock_conv0_fprop: outside the op's envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x && w && a && d && y, "gblock_conv0_fprop: x, w, a, d, y must not be NULL");
    LVG_REQUIRE(num_sms() <= kMaxSms, "gblock_conv0_fprop: more than %d SMs", kMaxSms);
    const FpropRooms r = fprop_rooms(sh, num_sms());
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= r.total(), "gblock_conv0_fprop: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    IgemmJob j = fprop_job(sh, x, w, y);
    j.in_scale = a; j.out_scale = d;
    j.bias = b; j.act = act; j.alpha = alpha; j.gain = gain; j.clamp = clamp;
    const int rc = run_igemm(j, workspace, r.job, s);
    if (rc || !sumsq) return rc;
    return sumsq_of(y, dtype, (int64_t)n * cout * sh.thw(), reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + r.job), sumsq, s);
}

extern "C" int lvg_gblock_conv0_backward(const void* x, const void* w, const float* a, const float* d, const float* b, const void* y, const void* dy,
                                         void* dx, void* dw, float* da, float* dd, float* db, int dtype, int n, int cin, int cout, int t, int h, int wd,
                                         int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int act, float alpha, float gain, float clamp,
                                         void* workspace, int64_t workspace_bytes, void* stream)
{
    const ConvShape sh = conv0_shape(dtype, n, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w);
    if (!conv0_ok(sh, act)) {
        set_error("gblock_conv0_backward: outside the op's envelope");
        return LVG_UNSUPPORTED;
    }
    LVG_REQUIRE(x && w && a && d && y && dy && dx && da, "gblock_conv0_backward: x, w, a, d, y, dy, dx, da must not be NULL");
    const int64_t rr = rows_room(sh);
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= rr + backward_workspace(sh),
                "gblock_conv0_backward: workspace too small or misaligned");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    float* s1 = reinterpret_cast<float*>(ws);
    const int to = sh.to();
    const int64_t rows = (int64_t)n * cout * to, len = (int64_t)sh.ho() * sh.wo();
    {
        int64_t blocks = std::min<int64_t>(rows, (int64_t)num_sms() * 8);
        const RowArgs ra = {act, alpha, gain, gain != 0.f ? 1.f / gain : 0.f, clamp};
        const int es = dtype == LVG_F32 ? 4 : 2;
        const bool vec = aligned16(y) && aligned16(dy) && (len * es) % 16 == 0;
        if (dtype == LVG_F32) {
            if (vec) conv0_rows_kernel<float, 4><<<(unsigned)blocks, 256, 0, s>>>((const float*)dy, (const float*)y, b, d, s1, dd, rows, len, cout, to, ra);
            else conv0_rows_kernel<float, 1><<<(unsigned)blocks, 256, 0, s>>>((const float*)dy, (const float*)y, b, d, s1, dd, rows, len, cout, to, ra);
        } else {
            if (vec) conv0_rows_kernel<__half, 8><<<(unsigned)blocks, 256, 0, s>>>((const __half*)dy, (const __half*)y, b, d, s1, dd, rows, len, cout, to, ra);
            else conv0_rows_kernel<__half, 1><<<(unsigned)blocks, 256, 0, s>>>((const __half*)dy, (const __half*)y, b, d, s1, dd, rows, len, cout, to, ra);
        }
        LVG_LAUNCH_CHECK();
        if (db) {
            conv0_db_kernel<<<(unsigned)((cout + 255) / 256), 256, 0, s>>>(s1, db, n, cout, to);
            LVG_LAUNCH_CHECK();
        }
    }
    const ActGate gate = {y, act, alpha, gain, clamp};
    Backward bw;
    int rc = backward_dgrad(sh, dy, d, w, dx, ws + rr, workspace_bytes - rr, s, bw, &gate);
    if (rc) return rc;
    rc = modconv_rowdot(dx, x, a, da, dtype, (int64_t)n * cin * t, (int64_t)h * wd, s);
    if (rc) return rc;
    return dw ? backward_wgrad(sh, bw, x, dy, d, dw, a, nullptr, s) : LVG_OK;
}
