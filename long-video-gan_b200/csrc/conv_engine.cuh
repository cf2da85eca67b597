// Host interface of the convolution engine (conv_igemm.cu) for the fused ops that drive it (modconv.cu, sres_layer.cu,
// sres_dblock.cu), and the device helpers their re-tiling and row-dot kernels share with the engine's.
//
// A call is described once (ConvShape); each kernel launch of the forward kernel is a job (IgemmJob) derived from it by
// fprop_job / dgrad_job, which a caller changes only where its call differs (factors, a pre-tiled input). Every call that
// uses a workspace carves it from one rooms struct, whose total is also what its size query returns.
#pragma once

#include <cuda_bf16.h>

#include "common.cuh"

namespace lvg {

__device__ __forceinline__ unsigned short bf16_bits(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float bf16_val(unsigned short b) { return __uint_as_float((uint32_t)b << 16); }

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ void from_f32(float& o, float v) { o = v; }
__device__ __forceinline__ void from_f32(__half& o, float v) { o = __float2half_rn(v); }

inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
inline int64_t round256(int64_t b) { return (b + 255) / 256 * 256; }

// One convolution call: x [n][groups * cin][t][h][wd], w [groups * cout][cin][kt][kh][kw], zero padding, spatial stride.
struct ConvShape {
    int dtype, n, groups, cin, cout, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w, stride;

    int split() const { return dtype == LVG_F32 ? 1 : 0; }
    int taps() const { return kt * kh * kw; }
    int64_t inst() const { return (int64_t)n * groups; }
    int64_t thw() const { return (int64_t)t * h * wd; }
    int to() const { return t + 2 * pad_t - kt + 1; }      // stride-1 output extent
    int ho() const { return h + 2 * pad_h - kh + 1; }
    int wo() const { return wd + 2 * pad_w - kw + 1; }
    int hos() const { return (ho() - 1) / stride + 1; }    // strided output extent
    int wos() const { return (wo() - 1) / stride + 1; }
    bool empty() const { return to() < 1 || ho() < 1 || wo() < 1; }

    bool tileable() const;       // the engine's operand geometry exists (dtype, kernel extent, n, groups)
    bool fprop_ok() const;       // the forward kernel takes the call
    bool dgrad_ok() const;       // ... and its input gradient (padding <= k - 1)
    bool wgrad_ok() const;       // the weight-gradient kernel takes the call
};

// K-side geometry of one GEMM: `ck` contraction channels and `cm` output channels per group
struct Geometry {
    int cpad, cblk, nblk, nimg, kc, mt;
    int m64, a_img;              // 64-row mode, bytes of one weight image
    int64_t act_bytes, w_bytes;
};
Geometry geometry(int split, int64_t inst, int groups, int ck, int cm, int64_t thw, int taps);

// bias_act's gradient rule applied while a gradient dy is re-tiled: dy * G(y) with G decided from the layer's output y
// (same layout as dy) as bias_act's grad-1 kernel decides it: slope 1 or alpha (lrelu) by the sign of y, times gain, 0 where
// y is not inside (-clamp, clamp). act: 1 linear, 2 lrelu (the engine epilogue's codes); y == nullptr: no gate.
struct ActGate {
    const void* y;
    int act;
    float alpha, gain, clamp;
};

// One launch of the forward kernel: y = correlation of x with the weights, or the input gradient run as one.
struct IgemmJob {
    // input operand: x (or, x8_pre != nullptr, its re-tiled X8, which the job then does not read or write), in_scale
    // [inst][ck][t] multiplies x while it is re-tiled; x is an xin_h x xin_w image placed on every dil-th pixel of h x wd
    const void* x;
    const unsigned char* x8_pre;
    const float* in_scale;
    ActGate in_gate;             // (input gradients) dy re-tiled as dy * G(y) * in_scale
    int xin_h, xin_w, dil;
    // GEMM shape and padding: ck channels in, cm out, per group
    int dtype, n, groups, ck, cm, t, h, wd, kt, kh, kw, pad_t, pad_h, pad_w;
    // weight access: A[m][k][tap] = w[g * gs + m * sm + k * sk + (flip ? taps - 1 - tap : tap)]
    const void* w;
    int64_t gs, sm, sk;
    int flip;
    // epilogue: [bias, act(alpha), gain, clamp], out_scale [inst][cm][to] on the accumulators
    void* y;
    const float* bias;
    int act;
    float alpha, gain, clamp;
    const float* out_scale;
    int ostride;                 // only every ostride-th output row / column is stored
};
IgemmJob fprop_job(const ConvShape& s, const void* x, const void* w, void* y);
IgemmJob dgrad_job(const ConvShape& s, const void* dy, const void* w, void* dx);

// workspace of a job: [packed weights][X8 of the input, unless pre-tiled]
struct IgemmRooms {
    int64_t wp, x8;
    int64_t total() const { return wp + x8 + 256; }
};
IgemmRooms igemm_rooms(const IgemmJob& j);
int run_igemm(const IgemmJob& j, void* workspace, int64_t workspace_bytes, cudaStream_t s);

struct WgradPlan {
    int split, cpad_a, cpad_b, nt, ntiles, mt, nsplit;
    int ablk, khc, mrows;
    int nseg, seg_w[4], seg_x0[4], ps, rh, stages;
    int a_stage, b_stage, stage_bytes, tail_bytes;
    size_t smem;
    int64_t a_bytes, b_bytes, part_bytes, dw_elems;
};
WgradPlan wgrad_plan(const ConvShape& s, bool fold = true);

// what a weight-gradient call takes in place of re-tiling its operands: dy8_pre / x8_pre (then dy / x are not read), or
// the factors the re-tiling applies: x_scale [n][cin][t], dy_scale [n][cout][to]
struct WgradInputs {
    const unsigned char* dy8_pre;
    const unsigned char* x8_pre;
    const float* x_scale;
    const float* dy_scale;
    ActGate dy_gate;             // dy re-tiled as dy * G(y) * dy_scale
};

// workspace of a weight gradient: [dy8, unless pre-tiled][x8][fp32 partial sums]
struct WgradRooms {
    int64_t dy8, x8, part;
    int64_t total() const { return dy8 + x8 + part + 512; }
};
WgradRooms wgrad_rooms(const WgradPlan& q, bool dy8_pre);
int run_wgrad(const ConvShape& s, const void* x, const void* dy, void* dw, const WgradInputs& in, void* workspace, int64_t workspace_bytes,
              cudaStream_t st);

// Both gradients of one call on the engine, in two halves so that a caller's own pass can run between them.
// backward_dgrad writes dx = conv^T(d (.) dy, w) (d [n][cout][to] or nullptr); when shares_dy8(), d (.) dy is re-tiled once
// and backward_wgrad reads the same tiles. Workspace: [d dy re-tiled, when shared][rest: the input gradient's job, then the
// weight gradient's].
struct BackwardRooms {
    int64_t dy8, rest;
    int64_t x8;                  // where in rest the weight gradient re-tiles x
    int64_t total() const { return dy8 + rest; }
};
bool shares_dy8(const ConvShape& s);
BackwardRooms backward_rooms(const ConvShape& s, bool shared);
int64_t backward_workspace(const ConvShape& s);          // the largest of the layouts the call may take
struct Backward {
    const unsigned char* dy8;    // the shared tiles, or nullptr
    unsigned char* rest;
    int64_t rest_bytes;
    unsigned char* x8;           // where the weight gradient re-tiles x: a caller may build X8 there and pass it as x8_pre
    ActGate gate;                // the gate dy was re-tiled with (the weight gradient applies it too when it re-tiles dy itself)
};
// gate != nullptr: both gradients take dy * G(y) (bias_act's gradient) in place of dy, without it being written
int backward_dgrad(const ConvShape& s, const void* dy, const float* d, const void* w, void* dx, void* workspace, int64_t workspace_bytes,
                   cudaStream_t st, Backward& b, const ActGate* gate = nullptr);
int backward_wgrad(const ConvShape& s, const Backward& b, const void* x, const void* dy, const float* d, void* dw, const float* x_scale,
                   const unsigned char* x8_pre, cudaStream_t st);

// modconv.cu: the modulated convolution's envelope; r[row] = sum_i u[row][i] v[row][i], scale != nullptr: u[row][i] *=
// scale[row] in place
bool modconv_in_envelope(const ConvShape& s);
int modconv_rowdot(void* u, const void* v, const float* scale, float* r, int dtype, int64_t rows, int64_t len, cudaStream_t s);

}  // namespace lvg
