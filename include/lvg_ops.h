/*
 * lvg_ops.h -- C ABI of liblvg_ops.so, the sm_90a operator library behind the
 * torch_utils.ops drop-in (bias_act, upfirdn2d, filtered_lrelu, fma, and the
 * 1-D / 2-D / 3-D convolution engine behind conv2d_gradfix and conv_nd).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in _host;
 *   - the caller owns all buffers (outputs are allocated by the host side,
 *     e.g. torch.empty) -- the library never allocates device memory that
 *     outlives a call, and keeps no mutable global device state, so calls are
 *     safe from any thread on any stream;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *     calls only enqueue work and never synchronise;
 *   - strides are in ELEMENTS, shapes are [N, C, H, W] order;
 *   - return 0 = launched, LVG_UNSUPPORTED (-1) = no kernel for this
 *     configuration (the caller may compose other entry points, mirroring the
 *     reference plugin's return code, filtered_lrelu.cpp:53-57), >0 = argument
 *     or CUDA error; lvg_last_error() then describes it (thread local).
 *
 * Each entry point names the reference plugin function it replaces
 * (paths relative to the NVlabs/long-video-gan tree).
 */
#ifndef LVG_OPS_H_
#define LVG_OPS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LVG_ABI_VERSION 2

#define LVG_OK            0
#define LVG_UNSUPPORTED (-1)
#define LVG_ERR_ARG       1
#define LVG_ERR_CUDA      2

/* element types */
#define LVG_F32 0
#define LVG_F16 1
#define LVG_F64 2

/* activation codes: same numbering as `cuda_idx` in torch_utils/ops/bias_act.py:21-31 */
#define LVG_ACT_LINEAR   1
#define LVG_ACT_RELU     2
#define LVG_ACT_LRELU    3
#define LVG_ACT_TANH     4
#define LVG_ACT_SIGMOID  5
#define LVG_ACT_ELU      6
#define LVG_ACT_SELU     7
#define LVG_ACT_SOFTPLUS 8
#define LVG_ACT_SWISH    9

int         lvg_abi_version(void);
const char* lvg_last_error(void);
/* compile-time facts about the build: "sm_90a;..." */
const char* lvg_build_info(void);
/* number of kernels this library has launched in the calling process so far */
int64_t     lvg_launch_count(void);

/*
 * bias_act -- replaces bias_act_plugin.bias_act (torch_utils/ops/bias_act.cpp:32-90,
 * kernel bias_act.cu:23-147).
 *   grad = 0: y = clamp(act(x + b) * gain)
 *   grad = 1: y = x * gain * act'(.)   , zero where yref is outside (-clamp, clamp)
 *   grad = 2: y = x * dy * gain * act''(.), same masking
 * x, xref, yref, dy, y are dense buffers of n elements in one common layout;
 * the bias of element i is b[(i / step_b) % size_b]. NULL = operand absent.
 * clamp < 0 disables clamping.
 */
int lvg_bias_act(const void* x, const void* b, const void* xref, const void* yref,
                 const void* dy, void* y, int dtype, int64_t n, int64_t size_b,
                 int64_t step_b, int grad, int act, float alpha, float gain,
                 float clamp, void* stream);

/*
 * bias_act backward with the bias-gradient reduction fused in: as grad = 1
 * above, and additionally db[c] += sum of y over all elements whose bias index
 * is c (fp32 accumulators, db_f32 has size_b floats and must be zeroed by the
 * caller). Saves the extra read of dx that `dx.sum(...)` costs
 * (torch_utils/ops/bias_act.py:169-170).
 */
int lvg_bias_act_grad_db(const void* dy_in, const void* b, const void* xref,
                         const void* yref, void* dx, float* db_f32, int dtype,
                         int64_t n, int64_t size_b, int64_t step_b, int act,
                         float alpha, float gain, float clamp, void* stream);
/*
 * relu / lrelu with 2-bit codes instead of a saved output. The gradient of these activations depends on the
 * forward output only through "was it positive" and "was it saturated by the clamp"; the forward pass can
 * emit exactly those two bits per element (bit 0 = not positive, bit 1 = clamped) and the backward pass then
 * reads dy + codes (2 n s + n / 4 bytes) instead of dy + y (3 n s) -- same results as lvg_bias_act(grad = 1) /
 * lvg_bias_act_grad_db with yref = y (the reference always re-reads y: bias_act.py:160-172, bias_act.cu:60-118).
 * The codes buffer is opaque (tile-local word order of the kernels), 8-byte aligned, lvg_bias_act_codes_bytes(dtype, n)
 * bytes long (about n / 4), and only meaningful to lvg_bias_act_bwd_codes for a dy with the memory layout of x.
 * fwd: y and codes from x (+ b). bwd: dx from dy and codes; db_f32 != NULL also accumulates the bias gradient
 * (zero-initialised fp32 [size_b], bias along a non-contiguous dimension). Returns -1 when the activation is not
 * relu / lrelu, the type not fp32 / fp16, n not a multiple of the 16-byte pack or an operand unaligned.
 */
int lvg_bias_act_fwd_codes(const void* x, const void* b, void* y, void* codes, int dtype, int64_t n,
                           int64_t size_b, int64_t step_b, int act, float alpha, float gain, float clamp,
                           void* stream);
int lvg_bias_act_bwd_codes(const void* dy, const void* codes, void* dx, float* db_f32, int dtype, int64_t n,
                           int64_t size_b, int64_t step_b, int act, float alpha, float gain, float clamp,
                           void* stream);
int64_t lvg_bias_act_codes_bytes(int dtype, int64_t n);

/*
 * upfirdn2d -- replaces upfirdn2d_plugin.upfirdn2d (torch_utils/ops/upfirdn2d.cpp:16-98,
 * kernels upfirdn2d.cu:29-200). Full 2-D filter f[fh][fw] (float32, element
 * strides f_stride_y / f_stride_x). Output size per axis:
 *   out = (in * up + pad0 + pad1 - ftaps + down) / down      (upfirdn2d.cpp:35-36)
 * so y_shape carries the caller's choice of pad1. Any x / y strides.
 */
int lvg_upfirdn2d(const void* x, const float* f, void* y, int dtype,
                  const int64_t x_shape[4], const int64_t x_stride[4],
                  const int64_t y_shape[4], const int64_t y_stride[4],
                  int fw, int fh, int64_t f_stride_x, int64_t f_stride_y,
                  int upx, int upy, int downx, int downy, int padx0, int pady0,
                  int flip, float gain, void* stream);

/*
 * Separable upfirdn2d in ONE launch: horizontal pass with fx[fw], vertical
 * pass with fy[fh], the intermediate stays in shared memory. Replaces the two
 * chained plugin calls of torch_utils/ops/upfirdn2d.py:244-245 (and their HBM
 * round trip). fx == NULL or fy == NULL means "no filter along that axis"
 * (1 tap of weight 1). `gain` is applied once.
 * Returns LVG_UNSUPPORTED for shapes the tiled kernel does not cover
 * (caller then issues two lvg_upfirdn2d calls).
 */
int lvg_upfirdn2d_sep(const void* x, const float* fx, const float* fy, void* y,
                      int dtype, const int64_t x_shape[4], const int64_t x_stride[4],
                      const int64_t y_shape[4], const int64_t y_stride[4],
                      int fw, int fh, int upx, int upy, int downx, int downy,
                      int padx0, int pady0, int flip, float gain, void* stream);

/*
 * filtered_lrelu -- replaces filtered_lrelu_plugin.filtered_lrelu
 * (torch_utils/ops/filtered_lrelu.cpp:16-209, kernel filtered_lrelu.cu:139-1099):
 *   y = downfir( clamp( lrelu( upfir(x + b) * up^2 * gain ) ) )
 * fu / fd: float32, separable when f?_h == 0 (f?_w taps used on both axes),
 * else full [f?_h][f?_w] row-major. Sign tensor: uint8 [N][C][s_h][s_wbytes],
 * 2 bits per up-sampled sample, 4 samples per byte along x (bit0 = negative,
 * bit1 = clamped; filtered_lrelu.cu:494-519). Exactly one of the modes:
 *   write_signs != 0 : so written (forward with gradients)
 *   si != NULL       : signs read at offset (sx, sy) instead of evaluating lrelu/clamp (backward)
 *   neither          : plain forward
 * Returns LVG_UNSUPPORTED when no fused kernel covers (up, down, filter sizes),
 * and for the resampling configurations (up or down > 1) when slope > 1.
 * In read mode those configurations also need s_wbytes % 4 == 0 and si on a
 * 4-byte boundary (LVG_ERR_ARG otherwise); 1x1 filters take any slope and rows.
 */
int lvg_filtered_lrelu(const void* x, const float* fu, const float* fd, const void* b,
                       const uint8_t* si, void* y, uint8_t* so, int dtype,
                       const int64_t x_shape[4], const int64_t x_stride[4],
                       const int64_t y_shape[4], const int64_t y_stride[4],
                       int fu_w, int fu_h, int fd_w, int fd_h, int up, int down,
                       int px0, int py0, int s_h, int s_wbytes, int sx, int sy,
                       float gain, float slope, float clamp, int flip,
                       int write_signs, void* stream);

/* 0 if lvg_filtered_lrelu has a fused kernel for this configuration, else LVG_UNSUPPORTED */
int lvg_filtered_lrelu_supported(int dtype, int fu_w, int fu_h, int fd_w, int fd_h,
                                 int up, int down);

/*
 * In-place gain * lrelu * clamp with sign write / read -- replaces
 * filtered_lrelu_plugin.filtered_lrelu_act_ (filtered_lrelu.cpp:213-290,
 * kernel filtered_lrelu.cu:1105-1211). x is modified in place.
 */
int lvg_filtered_lrelu_act(void* x, const uint8_t* si, uint8_t* so, int dtype,
                           const int64_t x_shape[4], const int64_t x_stride[4],
                           int s_h, int s_wbytes, int sx, int sy, float gain,
                           float slope, float clamp, int write_signs, void* stream);

/*
 * fma -- out = a * b + c with numpy-style broadcasting (torch_utils/ops/fma.py:15-25).
 * All operands are described on the common broadcast shape (rank <= 6):
 * a stride of 0 marks a broadcast dimension. out is dense in `shape` order.
 */
int lvg_fma(const void* a, const void* b, const void* c, void* out, int dtype,
            int rank, const int64_t shape[6], const int64_t a_stride[6],
            const int64_t b_stride[6], const int64_t c_stride[6], void* stream);

/*
 * Grouped 1-D / 2-D / 3-D convolution (cross-correlation) on Hopper tensor cores (wgmma), TMA-fed (csrc/conv_igemm.cu): one
 * engine for conv2d_gradfix.conv2d / conv_transpose2d (conv2d_gradfix.py:37-45), the F.conv3d calls of the low-res
 * networks (generator_lres.py:119,578; discriminator_lres.py:172) and the F.conv1d calls of the low-res discriminator
 * (discriminator_lres.py:108-127).
 *   x [N][G*Cin][T][H][W]   w [G*Cout][Cin][kt][kh][kw]   y [N][G*Cout][To][Ho][Wo]      (dense; 2-D: T = kt = 1)
 * kh*kw <= 9, kt <= 7; `stride` (1..4) applies to H and W (T: 1) -- a strided forward pass computes the stride-1 result and
 * stores every stride-th row / column, its gradients spread dy over that lattice. dtype LVG_F16: fp16 operands, fp32 accumulation, fp16 result. dtype LVG_F32: operands
 * split into bf16 hi + lo halves, hi*hi + lo*hi + hi*lo accumulated in fp32 (fp32-grade result, relative error
 * ~2^-16; the reference runs these layers in strict fp32, train_lres.py:269). Optional fused epilogue on fprop:
 * act 0 = none, 1 = (y + bias[co]) * gain clamped, 2 = lrelu(y + bias[co], alpha) * gain clamped (bias_act semantics,
 * bias_act.py:52-86; clamp < 0 = none; bias indexed g*Cout + co, may be NULL).
 * dgrad / wgrad: gradients with respect to x / w; their argument lists describe the FORWARD convolution.
 * `workspace`: lvg_convnd_workspace (fprop, dgrad) or lvg_convnd_wgrad_workspace bytes, 16-byte aligned, holds the
 * re-tiled operands (and the split-K partial sums of wgrad). Return LVG_UNSUPPORTED (-1 from the size queries) outside
 * the envelope.
 */
int64_t lvg_convnd_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                             int kt, int kh, int kw, int pad_t, int pad_h, int pad_w);
int lvg_convnd_fprop(const void* x, const void* w, void* y, int dtype, int n, int groups, int cin, int cout,
                     int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride,
                     const float* bias, int act, float alpha, float gain, float clamp,
                     void* workspace, int64_t workspace_bytes, void* stream);
int lvg_convnd_dgrad(const void* dy, const void* w, void* dx, int dtype, int n, int groups, int cin, int cout,
                     int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride,
                     void* workspace, int64_t workspace_bytes, void* stream);
int64_t lvg_convnd_wgrad_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                                   int kt, int kh, int kw, int pad_t, int pad_h, int pad_w);
int lvg_convnd_wgrad(const void* x, const void* dy, void* dw, int dtype, int n, int groups, int cin, int cout,
                     int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride,
                     void* workspace, int64_t workspace_bytes, void* stream);
/*
 * Introspection: the tiling lvg_convnd_fprop (mode 0) / lvg_convnd_dgrad (mode 1) launches with, as 48 ints -- wgroups, cout
 * (rows of the GEMM), mt, kc, nblk, nimg, lo_blk, to, ho, wo, kt, kh, kw, pad_t, pad_h, pad_w, tt, th, wt, wtb, thb, frame_px,
 * ncols, tiles_x, tiles_y, tiles_t, total_tiles, ks, stages, a_resident, a_stage, b_step, b_bytes, b_box,
 * stage_bytes, ostride, hos, wos, 0..., [47] = 1 when the call takes the streaming 1x1x1 kernels instead -- host arithmetic only
 * (no device needed): tests/test_igemm_emul.py replays the kernel's addressing with it on the CPU. The argument list describes
 * the FORWARD convolution in both modes.
 */
int lvg_convnd_plan(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                    int pad_t, int pad_h, int pad_w, int stride, int* out, int out_len);
/*
 * Introspection: the epilogue of the launch lvg_convnd_plan describes, as 4 ints -- [0] 1 when adjacent accumulator
 * columns are stored as one 8-byte fp32 / 4-byte half2 pair (unit stride, even tile widths, output width and channel
 * stride; the launch also needs y aligned to a pair), 0 for one store per element, -1 when the call takes the streaming
 * 1x1x1 kernels; [1] stages of the operand ring (= lvg_convnd_plan's); [2] dynamic shared memory bytes of the launch;
 * [3] static shared memory bytes of the column map. Host arithmetic only, same arguments as lvg_convnd_plan.
 */
int lvg_convnd_epilogue_plan(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh,
                             int kw, int pad_t, int pad_h, int pad_w, int stride, int* out, int out_len);
/*
 * Introspection: the kernels a call takes -- mode 0 forward (`epilogue` != 0: with bias / act / gain / clamp), 1 input
 * gradient, 2 weight gradient -> 0 the implicit-GEMM engine, 1 the streaming SIMT kernels for few-channel fp32 1x1x1
 * layers, 2 the pointwise wgmma kernels for every other 1x1x1 forward / input gradient (stride 1, no padding, groups 1,
 * T*H*W a multiple of 4 (fp32) / 8 (fp16)); LVG_UNSUPPORTED outside the envelope. Host arithmetic only; tensors are
 * taken to be 16-byte aligned (route 2 runs on the engine for a misaligned one). LVG_CONV_PW_TC=0 turns route 2 off.
 */
int lvg_convnd_route(int mode, int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                     int pad_t, int pad_h, int pad_w, int stride, int epilogue);
/*
 * Introspection: the tiling lvg_convnd_wgrad launches with, as 32 ints -- split, cpad_a, cpad_b, nt, ntiles, mt, nsplit,
 * ablk, khc, nseg, ps, rh, stages, a_stage, b_stage, stage_bytes, tail_bytes, smem, seg_w[4], seg_x0[4], 0, mrows, 0... --
 * host arithmetic only (no device needed): tests/test_wgrad_emul.py replays the kernel's addressing with it on the CPU.
 */
int lvg_convnd_wgrad_plan(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                          int pad_t, int pad_h, int pad_w, int* out, int out_len);
/*
 * Introspection: the K steps lvg_convnd_wgrad takes over one stage of `rows` (1..rh) dy rows of column segment `seg`:
 * out[0] = steps, then per step the pixel offset of its first 8-pixel group and the distance to its second. Host
 * arithmetic only: tests/test_wgrad_ksteps_emul.py replays them on the CPU.
 */
int lvg_convnd_wgrad_ksteps(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                            int pad_t, int pad_h, int pad_w, int rows, int seg, int* out, int out_len);
/*
 * Both gradients of one convolution call (what autograd asks of F.conv3d / conv2d_gradfix in a first-order backward pass,
 * conv2d_gradfix.py:118-141): dx as lvg_convnd_dgrad, dw as lvg_convnd_wgrad, with dy re-tiled ONCE for the two kernels
 * (the separate entry points re-tile it once each). Argument list = the FORWARD convolution; `workspace`:
 * lvg_convnd_backward_workspace bytes.
 */
int64_t lvg_convnd_backward_workspace(int dtype, int n, int groups, int cin, int cout, int t, int h, int wd,
                                      int kt, int kh, int kw, int pad_t, int pad_h, int pad_w);
int lvg_convnd_backward(const void* x, const void* dy, const void* w, void* dx, void* dw, int dtype, int n, int groups,
                        int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w,
                        int stride, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Modulated convolution with one shared weight (groups = 1, stride 1), fp16 or fp32 (bf16 hi/lo split):
 *   y[n][co][ot] = d[n][co][ot] * sum_{ci,taps} w[co][ci][taps] * a[n][ci][t] * x[n][ci][t][...]
 * -- the style modulation / demodulation of modulated_conv2d (generator_sres.py:28-67, as N*T samples of 2-D images) and
 * temporal_modulated_conv3d (generator_lres.py:83-125) without per-sample weights. a [n][cin][t] (required) scales x while
 * it is re-tiled, d [n][cout][to] (NULL = none) the fp32 accumulators; t = 1 for 2-D. Argument order as lvg_convnd_fprop
 * with groups = 1. `workspace`: lvg_modconv_workspace bytes (forward and backward), 16-byte aligned; -1 / LVG_UNSUPPORTED
 * outside the envelope of lvg_convnd_backward (kh * kw <= 9, kw <= 3, kt <= 7, 0 <= pad <= k - 1).
 * Backward: dx = a * conv^T(d * dy, w), dw = sum_n conv_w(a * x, d * dy) (NULL = skipped), da[n][ci][t] = sum_hw
 * conv^T(d * dy, w) * x (NULL = skipped), dyy[n][co][ot] = sum_hw dy * y (NULL = skipped; needs y and d; the gradient of d
 * is dyy / d). d * dy is re-tiled once for both gradients when cout < 128 or a multiple of 128.
 */
int64_t lvg_modconv_workspace(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                              int pad_t, int pad_h, int pad_w);
int lvg_modconv_fprop(const void* x, const void* w, const float* a, const float* d, void* y, int dtype, int n, int cin,
                      int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w,
                      void* workspace, int64_t workspace_bytes, void* stream);
int lvg_modconv_backward(const void* x, const void* w, const float* a, const float* d, const void* y, const void* dy,
                         void* dx, void* dw, float* da, float* dyy, int dtype, int n, int cin, int cout, int t, int h,
                         int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, void* workspace,
                         int64_t workspace_bytes, void* stream);

/*
 * Depthwise long FIR along the last axis (cross-correlation, no padding), fp32:
 *   y[n][g][t] = sum_k w[g][k] * x[n][g][t + k],   x [n][groups][lin], w [groups][k], y [n][groups][lin - k + 1]
 * -- BlurredNoise.blur of the low-res generator: F.conv1d(noise, blur_filters [128, 1, 5000], groups = 128)
 * (model/generator_lres.py:378-387). Leading zero taps of each filter are skipped. `workspace`:
 * lvg_fir1d_depthwise_workspace(groups) bytes. Forward only (the input is noise, the filters are buffers).
 */
int64_t lvg_fir1d_depthwise_workspace(int groups);
int lvg_fir1d_depthwise(const float* x, const float* w, float* y, int n, int groups, int lin, int k,
                        void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Separable 4-tap FIR over the T, H, W axes of a contiguous NCTHW tensor (fp32 or fp16, fp32 accumulation), and its exact
 * adjoint. The operator P maps x [n][c][t_in][h_in][w_in] to y [n][c][t_out][h_out][w_out]; per axis, filt = 0 copies
 * (in == out) and filt = 1 computes  out[m] = sum_j f[3 - j] * in[step * m + off + j]  (step 1 or 2, zero outside the
 * input) -- Downsample3d's [1,3,3,1]/8 filter (discriminator_lres.py:186-213) at full rate or with step 2. fold = 1 stores
 * the T axis of the filtered side (t_out even) as two phase blocks of channels: [n][2c][t_out / 2], t = 2 t' + p -> channel
 * p * c + ci. f: 4 fp32 taps on the device. lvg_fir3d_adjoint takes the same arguments describing P and computes
 * x' = P^T y' (y' laid out as P's output, x' as P's input).
 */
int lvg_fir3d(const void* x, const float* f, void* y, int dtype, int n, int c, int t_in, int h_in, int w_in, int t_out,
              int h_out, int w_out, int filt_t, int filt_h, int filt_w, int step_t, int step_h, int step_w, int off_t,
              int off_h, int off_w, int fold, void* stream);
int lvg_fir3d_adjoint(const void* x, const float* f, void* y, int dtype, int n, int c, int t_in, int h_in, int w_in,
                      int t_out, int h_out, int w_out, int filt_t, int filt_h, int filt_w, int step_t, int step_h,
                      int step_w, int off_t, int off_h, int off_w, int fold, void* stream);

/*
 * Input augmentation of the low-res discriminator, fp32: DiffAugment's color, translation and cutout steps and the
 * temporal-scale augmentation of LowResVideoGAN.run_D (video_gan_lres.py:237-266, diff_augment.py) as one per-sample
 * affine map x [n][c][t_in][h][w] -> y [n][c][t_out][h][w] (DESIGN.md 7d). params: fp32 [n][12] on the device, per sample
 *   beta, sigma, kappa, dh, dw, r0, r1, c0, c1, r, L, off
 * (brightness, saturation, contrast; integer translation; cutout rows [r0, r1] x columns [c0, c1] of the translated frame,
 * empty when r1 < r0; output frame t reads frame u = t + off of the interpolated clip of length L, 2-tap
 * align_corners=False interpolation with reciprocal scale r, zero outside [0, L)). The integers are stored exactly in
 * fp32. flags: LVG_VIDEO_AUGMENT_LINEAR drops beta (the linear part of the map). lvg_video_augment_adjoint computes
 * dx = A^T dy of the linear part, the same arguments describing the forward map. `workspace`:
 * lvg_video_augment_workspace bytes (per-CTA partial sums of the per-sample means, folded in a fixed order: results are
 * bitwise reproducible; no atomics). Two kernel launches per call. LVG_UNSUPPORTED for c > 4. L is read on the device,
 * so the caller keeps L >= 1 (the draw of the scale does: LowResVideoGAN's F.interpolate fails for an empty clip);
 * frames outside [0, L) are zero for any L.
 */
#define LVG_VIDEO_AUGMENT_LINEAR 1
int64_t lvg_video_augment_workspace(int n, int c, int t_in, int h, int w, int t_out);
int lvg_video_augment(const float* x, const float* params, float* y, void* workspace, int n, int c, int t_in, int h, int w,
                      int t_out, int flags, void* stream);
int lvg_video_augment_adjoint(const float* dy, const float* params, float* dx, void* workspace, int n, int c, int t_in,
                              int h, int w, int t_out, void* stream);

/*
 * ADA's AugmentPipe (ada_augment.py:115-439) of the super-res step without imgfilter and cutout, fp32, c = 3: one affine map
 * per sample of x [n][c][t][h][w] (DESIGN.md 7e). With LVG_AUGMENT_PIPE_GEOM
 *   y = C[:3,:3] . downsample2d(grid_sample(upsample2d(reflect_pad(x, margins), f), affine_grid(theta)), f) + C[:3,3] + sigma noise
 * (upsample2d up = 2; grid of (2h + 12) x (2w + 12), bilinear, zeros, align_corners = False; downsample2d down = 2,
 * padding -6, flip_filter), without it y = C[:3,:3] x + C[:3,3] + sigma noise, mixing the 3 channels of a frame per pixel.
 * params: fp32 [n][LVG_AUGMENT_PIPE_NPAR] on the device, per sample
 *   mx0, my0, mx1, my1, theta[2][3], C[3][4], sigma
 * (the batch-wide reflect-pad margins, integers stored exactly, 0 <= margin <= size - 1; affine_grid's theta; the colour
 * matrix; the noise scale). filter: the ntaps taps of Hz_geom on the device. noise: [n][c][t][h][w] or NULL (no noise
 * term). LVG_AUGMENT_PIPE_LINEAR drops C[:3,3] and the noise (the linear part A). lvg_augment_pipe_adjoint computes
 * dx = A^T dy, the same arguments describing the forward map; with GEOM it needs `workspace` of
 * lvg_augment_pipe_workspace bytes (D^T C^T dy on the sampled grid). One kernel launch per call, two for the geometric
 * adjoint; no atomics, results are bitwise reproducible. LVG_UNSUPPORTED for c != 3 or ntaps != 12.
 */
#define LVG_AUGMENT_PIPE_NPAR 23
#define LVG_AUGMENT_PIPE_GEOM 1
#define LVG_AUGMENT_PIPE_LINEAR 2
int64_t lvg_augment_pipe_workspace(int n, int c, int t, int h, int w, int flags);
int lvg_augment_pipe(const float* x, const float* params, const float* filter, int ntaps, const float* noise, float* y, int n,
                     int c, int t, int h, int w, int flags, void* stream);
int lvg_augment_pipe_adjoint(const float* dy, const float* params, const float* filter, int ntaps, float* dx, void* workspace,
                             int n, int c, int t, int h, int w, int flags, void* stream);

/*
 * Tail of the low-res generator's residual block (Synthesis3dResBlock.forward, generator_lres.py:577-589), fp32 or fp16
 * storage with fp32 arithmetic, as one op over s, h [n][c][t][h][w] -> z [n][c][t_out][h_out][w_out] (DESIGN.md 7f):
 *   m = (s + h) sqrt(1/2);  u = crop_T(U_T m);  v = crop_HW(U_HW u);  z = bias_act(v, b, act, alpha, gain, clamp)
 * U_T (flag LVG_GBLOCK_TAIL_TUP) / U_HW (LVG_GBLOCK_TAIL_SUP): 2x upsampling with [1,3,3,1]/8 at gain 2 per axis and
 * padding (2, 1), as upfirdn2d.upsample2d; without the flag the axis is copied. The crops are center_crop's: offset
 * (size - out) / 2, 1 <= out <= size on every axis. b: fp32 [c] or NULL. act: LVG_ACT_LRELU or LVG_ACT_LINEAR
 * (LVG_UNSUPPORTED otherwise); clamp < 0 = none. codes (NULL = none): the 2-bit codes of z in lvg_bias_act_fwd_codes'
 * layout, lvg_bias_act_codes_bytes(dtype, numel(z)) bytes. s, h and z are dense and 16-byte (fp32) / 8-byte (fp16)
 * aligned. One kernel launch.
 * lvg_gblock_tail_adjoint: from dz and the codes, dv = the bias_act gradient, db[c] = sum of dv over n, t, h, w (fp32, a
 * fixed summation order: bitwise reproducible, no atomics) and dm = sqrt(1/2) * the transposed upsamplings and crops
 * applied to dv -- the gradient of both s and h. alpha and gain as in the forward call. `workspace`:
 * lvg_gblock_tail_workspace bytes (per-CTA partial sums of db). Two kernel launches. The size query returns -1 for shapes
 * outside the envelope (crops larger than the axis, a w_out row of dv that does not fit the adjoint's shared-memory tile).
 */
#define LVG_GBLOCK_TAIL_TUP 1
#define LVG_GBLOCK_TAIL_SUP 2
int64_t lvg_gblock_tail_workspace(int n, int c, int t, int h, int w, int t_out, int h_out, int w_out, int flags);
int lvg_gblock_tail(const void* s, const void* h, const float* b, void* z, uint8_t* codes, int dtype, int n, int c, int t,
                    int hh, int ww, int t_out, int h_out, int w_out, int flags, int act, float alpha, float gain, float clamp,
                    void* stream);
int lvg_gblock_tail_adjoint(const void* dz, const uint8_t* codes, void* dm, float* db, void* workspace, int64_t workspace_bytes,
                            int dtype, int n, int c, int t, int hh, int ww, int t_out, int h_out, int w_out, int flags, int act,
                            float alpha, float gain, void* stream);

/*
 * Tail of the low-res discriminator's residual block (DiscriminatorBlock.forward after conv_1's convolution,
 * discriminator_lres.py:321-333, 169-179, 197-213), fp32 or fp16 storage with fp32 arithmetic, as one op over
 * y [n][c][t][h][w] -> z [n][c][t_out][h_out][w_out] (DESIGN.md 7g):
 *   z = scale * (bias_act(P y, b, act, alpha, gain, clamp) + s)
 * P: per axis a copy or Downsample3d's filter out[m] = sum_j f[3 - j] * in[2 m - 1 + j] (zero outside; the extent must be
 * even, the output extent is half of it) -- lvg_fir3d's operator with (filt, step, off) = (1, 2, -1) -- on T with
 * LVG_DBLOCK_TAIL_TDOWN and on H and W with LVG_DBLOCK_TAIL_SDOWN. With LVG_DBLOCK_TAIL_MERGE scale = sqrt(1/2) and
 * s [n][c][t_out][h_out][w_out] (NULL = zero) is the skip tensor; without it scale = 1 and s must be NULL. bias_act's
 * output is rounded to the storage type before s is added (as the composition stores it); read mode rounds only its
 * result. f: 4 fp32 taps on the device, NULL allowed where no axis is filtered. b: fp32 [c] or NULL. act: LVG_ACT_LRELU or LVG_ACT_LINEAR (LVG_UNSUPPORTED otherwise); clamp < 0 = none.
 * mode:
 *   LVG_DBLOCK_TAIL_NONE   z only; codes must be NULL.
 *   LVG_DBLOCK_TAIL_WRITE  z and the 2-bit codes of every output (bit 0: bias_act's stored value is not positive, bit 1: it
 *                          is clamped, both evaluated as bias_act evaluates them): lvg_dblock_tail_codes_bytes bytes, one
 *                          byte per 4 consecutive outputs along W (output k of the group in bits 2k, 2k + 1), rows padded
 *                          to ceil(w_out / 4) bytes, rows in z's order.
 *   LVG_DBLOCK_TAIL_READ   codes are an input: z = scale * (G (P y + b) + s) with G = gain, gain * alpha or 0 (clamped) per
 *                          output, for arbitrary y, b, s: the linear map that is the adjoint's backward.
 * One kernel launch.
 * lvg_dblock_tail_adjoint: from dz [n][c][t_out][h_out][w_out] and the codes, dv = scale * G dz, dy = P^T dv
 * [n][c][t][h][w], ds = scale * dz (NULL = not wanted) and db[c] = sum of dv over n, t, h, w (fp32). db is summed from one
 * partial per CTA in `workspace` (lvg_dblock_tail_workspace bytes), folded by a second kernel in a fixed order; the
 * partition depends on the shape only and there are no atomics, so every result is bitwise reproducible. alpha and gain
 * as in the forward call. Two kernel launches. Both size queries return -1 for shapes outside the envelope (an odd extent
 * on a filtered axis, more than 65535 tiles of 8 x 32 per plane, n * c >= 2^31); such calls return LVG_UNSUPPORTED.
 */
#define LVG_DBLOCK_TAIL_TDOWN 1
#define LVG_DBLOCK_TAIL_SDOWN 2
#define LVG_DBLOCK_TAIL_MERGE 4
#define LVG_DBLOCK_TAIL_NONE 0
#define LVG_DBLOCK_TAIL_WRITE 1
#define LVG_DBLOCK_TAIL_READ 2
int64_t lvg_dblock_tail_workspace(int n, int c, int t, int h, int w, int flags);
int64_t lvg_dblock_tail_codes_bytes(int n, int c, int t, int h, int w, int flags);
int lvg_dblock_tail(const void* y, const void* s, const float* b, const float* f, void* z, uint8_t* codes, int mode, int dtype,
                    int n, int c, int t, int h, int w, int flags, int act, float alpha, float gain, float clamp, void* stream);
int lvg_dblock_tail_adjoint(const void* dz, const uint8_t* codes, const float* f, void* dy, void* ds, float* db, void* workspace,
                            int64_t workspace_bytes, int dtype, int n, int c, int t, int h, int w, int flags, int act,
                            float alpha, float gain, void* stream);

/*
 * Input of a super-res generator layer (generator_sres.py: Generator.prep_cond, the concatenation in
 * SynthesisNetwork.forward and the cast in SynthesisLayer.forward) as one op, written in the layer's dtype (DESIGN.md 7h):
 *   z[n t + t', :c]               = z_dtype(x[n t + t'])                     (c = 0: no x)
 *   z[n t + t', c + k window + s] = z_dtype(A_H lr[n][k][t' + s] A_W^T)       k < c_lr, s < window
 * x: dense [n t][c][h_out][w_out] (x_dtype); lr: fp32 [n][c_lr][t_lr][h_lr][w_lr] with element strides lr_strides[5];
 * z: dense [n t][c + c_lr window][h_out][w_out], 16-byte aligned. A_H / A_W: the per-axis plan, LVG_SRES_COND_NPLAN ints
 * {out, px0, mhi, x0, up, down, pad0, zlen, shift, ntaps} (host memory): output index i reads the resampler output
 * m = x0 + clamp(i - px0, 0, mhi); that is gain * sum_k f[ntaps - 1 - k] * u[m down + k - pad0] with u the frame
 * upsampled by `up` (zeros inserted) and zero outside [0, zlen); sample v of the frame is low-res row / column
 * clamp(v - shift, 0, len - 1). ntaps = 0: an identity axis (up = down = 1, pad0 = 0, f NULL). f_h / f_w: the 1-D fp32
 * filters on the device, at most 64 taps. Values are accumulated in fp32 and rounded once.
 * mean_sq (NULL = not wanted): one fp32 on the device, the mean of the squares of the fp32 concatenation (x before any
 * cast, the conditioning before rounding), summed from one partial per CTA in `workspace` (lvg_sres_cond_workspace bytes)
 * by a second kernel in a fixed order: bitwise reproducible, no atomics. One kernel launch, two with mean_sq. The size
 * query returns -1 for shapes and plans it does not take (more than 64 taps, tap tables beyond shared memory, t +
 * window - 1 > t_lr, a z_dtype other than fp32 / fp16); such calls return LVG_UNSUPPORTED.
 */
#define LVG_SRES_COND_NPLAN 10
int64_t lvg_sres_cond_workspace(int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr, int z_dtype,
                                const int* plan_h, const int* plan_w);
int lvg_sres_cond(const void* x, const float* lr, const float* f_h, const float* f_w, void* z, float* mean_sq, void* workspace,
                  int64_t workspace_bytes, int x_dtype, int z_dtype, int n, int t, int c, int c_lr, int window, int t_lr,
                  int h_lr, int w_lr, const int64_t* lr_strides, const int* plan_h, const int* plan_w, float gain_h,
                  float gain_w, void* stream);

/*
 * A super-res generator layer's modulated convolution with its input built inside the convolution's re-tiling pass
 * (DESIGN.md 7j):  y = d (.) conv(a (.) z, w)  with  z = cat(x, cond(lr)).to(dtype)  as lvg_sres_cond defines it, z never
 * stored. x, lr, f_h, f_w, x_dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, lr_strides, plan_h, plan_w, gain_h, gain_w:
 * as lvg_sres_cond (dtype = its z_dtype, the layer's). The convolution as lvg_modconv_fprop with cin = c + c_lr window,
 * t = 1 and n t samples: w [cout][cin][kh][kw] (dtype), a fp32 [n t][cin], d fp32 [n t][cout] or NULL, y [n t][cout][ho][wo]
 * (dtype). Bit for bit lvg_modconv_fprop of lvg_sres_cond's z. mean_sq (NULL = not wanted): as lvg_sres_cond's, from
 * per-CTA partials folded in a fixed order (bitwise reproducible; not the same fold as lvg_sres_cond's). y NULL: mean_sq
 * alone, from the same pass without its stores (w, a unused), for callers whose factor a depends on the statistic.
 * lvg_sres_layer_backward: lvg_modconv_backward of that call with dx the gradient of x alone, written in x_dtype
 * (x_dtype(dtype(a dx')), the cast of z's gradient; NULL = not wanted), dw (NULL = not wanted), da [n t][cin] over all
 * channels, dyy (NULL = not wanted; needs y and d). One workspace size serves both calls; the size query returns -1 for
 * anything the kernels do not take, and the ops then return LVG_UNSUPPORTED.
 */
int64_t lvg_sres_layer_workspace(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                 const int* plan_h, const int* plan_w, int cout, int kh, int kw, int pad_h, int pad_w);
int lvg_sres_layer_fprop(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                         const float* d, void* y, float* mean_sq, int x_dtype, int dtype, int n, int t, int c, int c_lr,
                         int window, int t_lr, int h_lr, int w_lr, const int64_t* lr_strides, const int* plan_h,
                         const int* plan_w, float gain_h, float gain_w, int cout, int kh, int kw, int pad_h, int pad_w,
                         void* workspace, int64_t workspace_bytes, void* stream);
int lvg_sres_layer_backward(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                            const float* d, const void* y, const void* dy, void* dx, void* dw, float* da, float* dyy,
                            int x_dtype, int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                            const int64_t* lr_strides, const int* plan_h, const int* plan_w, float gain_h, float gain_w,
                            int cout, int kh, int kw, int pad_h, int pad_w, void* workspace, int64_t workspace_bytes,
                            void* stream);

/*
 * The super-res generator's ToRGB layer in one pass over its input (DESIGN.md 7k), on the CUDA cores:
 *   y = dtype(clamp(dtype(u) + b, +-clamp)),  u = sum_c w[o][c] r(a[c] z[c])  per pixel, o < cout = 3
 * with z = cat(x, cond(lr)).to(dtype) as lvg_sres_cond defines it, never stored, and r() the rounding of the convolution
 * engine's re-tiling pass (fp16 layers: fp16(a z); fp32 layers: a z in fp32); products accumulated in fp32. x, lr, f_h,
 * f_w, x_dtype, n, t, c, c_lr, window, t_lr, h_lr, w_lr, lr_strides, plan_h, plan_w, gain_h, gain_w: as lvg_sres_cond
 * (dtype = its z_dtype, the layer's). w [cout][cin] and b [cout] in dtype, cin = c + c_lr window; a fp32 [n t][cin];
 * y [n t][cout][h_out][w_out] (dtype). clamp >= 0 (infinity: none). mask (NULL = not wanted): [n t][h_out][w_out] bytes,
 * bit o set where output o was clamped (|dtype(u) + b| > clamp), which the backward needs. One kernel launch.
 * lvg_sres_torgb_backward, from the forward's mask and dy (dtype, y's shape): dy' = dy where not clamped, else 0;
 * dx' = dtype(w^T dy') per pixel; dx (NULL = not wanted) = x_dtype(dtype(a dx')) for the x channels; da [n t][cin] (fp32) =
 * sum over pixels of dx' z; dw [cout][cin] = dtype(sum over samples and pixels of dy' r(a z)) and db [cout] =
 * dtype(sum dy') (dtype; NULL = not wanted). Per-CTA partial sums in `workspace` (lvg_sres_torgb_workspace bytes), folded
 * by two more kernels in a fixed order: bitwise reproducible, no atomics. The forward needs no workspace. The size query
 * returns -1 for anything the kernels do not take (cout != 3, more than 1024 input channels, a conditioning
 * lvg_sres_cond_workspace rejects, an output wider than 2048 pixels); such calls return LVG_UNSUPPORTED.
 */
int64_t lvg_sres_torgb_workspace(int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                                 const int* plan_h, const int* plan_w, int cout);
int lvg_sres_torgb_fprop(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                         const void* b, void* y, unsigned char* mask, int x_dtype, int dtype, int n, int t, int c, int c_lr,
                         int window, int t_lr, int h_lr, int w_lr, const int64_t* lr_strides, const int* plan_h,
                         const int* plan_w, float gain_h, float gain_w, int cout, float clamp, void* stream);
int lvg_sres_torgb_backward(const void* x, const float* lr, const float* f_h, const float* f_w, const void* w, const float* a,
                            const unsigned char* mask, const void* dy, void* dx, void* dw, float* da, void* db, int x_dtype,
                            int dtype, int n, int t, int c, int c_lr, int window, int t_lr, int h_lr, int w_lr,
                            const int64_t* lr_strides, const int* plan_h, const int* plan_w, float gain_h, float gain_w,
                            int cout, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * The low-res generator's ToRGB layer in one pass over its input (DESIGN.md 7l), on the CUDA cores:
 *   y = dtype(clamp(dtype(u) + dtype(b), +-clamp)),  u = sum_c w[o][c] a[n][c][t] r(x[c])  per pixel, o < cout = 3
 * with r() the rounding of x.type(dtype) and the products accumulated in fp32. x: dense [n][cin][t][h][wd] in x_dtype
 * (fp16 / fp32), read in place; w fp32 [cout][cin] (the reference's weight / sqrt(cin)); a fp32 [n][cin][t] (style times
 * the magnitude-EMA gain); b fp32 [cout]; dtype (fp16 / fp32) the layer's. clamp < 0: none (bias_act's convention).
 * lvg_lres_torgb_fprop writes exactly one of y ([n][cout][t][h][wd], dtype) or u (same shape, fp32, before rounding,
 * bias and clamp). With sumsq (NULL = not wanted) it also writes the sum of r(x)^2 over the whole input to sumsq[0],
 * from per-CTA partials in `workspace` folded in a fixed order (one more launch). lvg_lres_torgb_finish then writes
 * y = dtype(clamp(dtype(gain[0] u) + dtype(b))) with the gain read from device memory (no host synchronisation).
 * lvg_lres_torgb_backward, from the forward's y and dy (dtype, y's shape): dy' = dy where -clamp < y < clamp, else 0;
 * dx (NULL = not wanted) = x_dtype(a w^T dy') per pixel; da [n][cin][t] = sum over the pixels of a plane of
 * sum_o w[o][c] dy'[o] r(x[c]); dw [cout][cin] (NULL = not wanted) = sum over planes of a times the same sums; db
 * [cout] (NULL = not wanted) = sum dy'; all fp32. Per-CTA partial sums in `workspace` (lvg_lres_torgb_workspace bytes,
 * which also covers the forward's sumsq), folded by two more kernels in a fixed order: bitwise reproducible, no
 * atomics. The size query returns -1 for anything the kernels do not take (cout != 3, a kernel other than 1 x 1 x 1
 * (kt, kh, kw), more than 512 input channels, a dtype other than fp16 / fp32); such calls return LVG_UNSUPPORTED.
 */
int64_t lvg_lres_torgb_workspace(int x_dtype, int dtype, int n, int cin, int t, int h, int wd, int cout, int kt, int kh, int kw);
int lvg_lres_torgb_fprop(const void* x, const float* w, const float* a, const float* b, void* y, float* u, float* sumsq,
                         int x_dtype, int dtype, int n, int cin, int t, int h, int wd, int cout, float clamp,
                         void* workspace, int64_t workspace_bytes, void* stream);
int lvg_lres_torgb_finish(const float* u, const float* gain, const float* b, void* y, int dtype, int n, int t, int h, int wd,
                          float clamp, void* stream);
int lvg_lres_torgb_backward(const void* x, const float* w, const float* a, const void* y, const void* dy, void* dx, float* dw,
                            float* da, float* db, int x_dtype, int dtype, int n, int cin, int t, int h, int wd, int cout,
                            float clamp, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * The first modulated convolution of the low-res generator's residual block with its bias_act (DESIGN.md 7m):
 *   y = clamp(act(d (.) conv(a (.) x, w) + b) * gain)
 * with x, w, a, d, the shapes and the padding as lvg_modconv_fprop (d required; the output keeps the input's frame count),
 * b fp32 [cout] or NULL, act 1 linear / 2 lrelu with alpha, gain and clamp (< 0: none) as lvg_convnd_fprop. The
 * pre-activation is never stored: the engine's epilogue applies d, the bias, the activation, the gain and the clamp.
 * sumsq (NULL = not wanted): sum of the squares of y as stored (rounded to dtype) in sumsq[0], fp32, from one more pass
 * over y (per-CTA partials over a fixed grid, folded in a fixed order: two more launches).
 * lvg_gblock_conv0_backward, from the forward's y and dy (y's dtype and shape), with dz = G(y) dy bias_act's gradient
 * (decided from y): dx (x's shape and dtype), dw (w's, NULL = not wanted), da [n][cin][t] as lvg_modconv_backward of dz;
 * dd [n][cout][t] (NULL = not wanted) = sum_hw dz (z(y) - b) / d with z(y) the pre-activation recovered from y; db [cout]
 * (NULL = not wanted) = sum dz over n, t, h, w in a fixed order; all fp32, bitwise reproducible. dz is never written: the
 * convolution gradients re-tile dy with G(y) and d. `workspace`: lvg_gblock_conv0_workspace bytes (forward and backward),
 * 16-byte aligned; -1 / LVG_UNSUPPORTED outside lvg_modconv_workspace's envelope or for an output frame count other than t.
 */
int64_t lvg_gblock_conv0_workspace(int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw,
                                   int pad_t, int pad_h, int pad_w);
int lvg_gblock_conv0_fprop(const void* x, const void* w, const float* a, const float* d, const float* b, void* y, float* sumsq,
                           int dtype, int n, int cin, int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t,
                           int pad_h, int pad_w, int act, float alpha, float gain, float clamp, void* workspace,
                           int64_t workspace_bytes, void* stream);
int lvg_gblock_conv0_backward(const void* x, const void* w, const float* a, const float* d, const float* b, const void* y,
                              const void* dy, void* dx, void* dw, float* da, float* dd, float* db, int dtype, int n, int cin,
                              int cout, int t, int h, int wd, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int act,
                              float alpha, float gain, float clamp, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Layers of a super-res discriminator block (discriminator_sres.py DiscriminatorBlock, architecture 'resnet'; DESIGN.md 7i).
 *
 * lvg_sres_dblock_conv1: conv1, y = bias_act(conv2d(upfirdn2d(x, f, padding 2), w, stride 2), bias, act, alpha, gain,
 * clamp) with f = outer(fy, fx) 4 x 4 (fx, fy: 4 fp32 taps each on the device; flip as upfirdn2d's flip_filter). The FIR
 * runs inside the convolution's re-tiling pass (fp32 accumulation, rounded once to fp16 or split once into bf16 halves); the
 * filtered image is never stored. x: dense fp16 / fp32 [n][cin][h][wd]; w: [cout][cin][3][3] in x's dtype; bias: fp32
 * [cout] or NULL; y: [n][cout][h / 2][wd / 2] rounded down plus one where odd ((h + 1 - 3) / 2 + 1). act: 0 none,
 * 1 linear, 2 lrelu, as lvg_convnd_fprop; clamp < 0: none. Two launches (re-tiling, convolution) plus the weight re-tiling.
 *
 * lvg_sres_dblock_skip: the skip with the residual merge, y = (W x + r) * rscale: a 1x1 convolution of the down-sampled
 * input x [n][cin][P] (w: [cout][cin]) on the pointwise wgmma kernels, the residual r [n][cout][P] (conv1's output, x's
 * dtype and layout) added to the fp32 accumulator and the sum scaled by rscale in the epilogue, one rounding to x's dtype.
 * x, r, y 16-byte aligned; P % 4 == 0 (fp32) or P % 8 == 0 (fp16).
 *
 * lvg_sres_dblock_conv1_backward: conv1's first-order backward from dy (the gradient of conv1's pre-activation, [n][cout]
 * [h / 2][wd / 2]): dhf = the gradient of the filtered image [n][cin][h + 1][wd + 1] (NULL = not wanted) as
 * lvg_convnd_dgrad computes it, and dw [cout][cin][3][3] (NULL = not wanted) from the weight-gradient kernel with its x
 * operand re-tiled straight from x by the FIR re-tiling pass: bit for bit lvg_convnd_wgrad of the filtered image that
 * pass computes, which is never stored in NCHW.
 *
 * lvg_sres_dblock_fir_adjoint_act: dz = G(h0) (.) FIR^T(dhf) for h0 [n][c][h][w] (conv0's output) and dhf [n][c][h + 1]
 * [w + 1]: the adjoint of upfirdn2d(., f, padding 2) (fp32, rounded once) times bias_act's first-order slope decided from h0
 * (act 1 linear / 2 lrelu, alpha, gain, clamp < 0: none); db (fp32 [c], NULL = not wanted) = the sum of the stored dz per
 * channel, per-CTA partials folded in a fixed order (no atomics, bitwise reproducible). Two launches.
 *
 * The size queries return -1 outside the envelope; the ops then return LVG_UNSUPPORTED.
 */
int64_t lvg_sres_dblock_conv1_workspace(int dtype, int n, int cin, int cout, int h, int wd);
int lvg_sres_dblock_conv1(const void* x, const float* fx, const float* fy, int flip, const void* w, const float* bias, void* y,
                          int dtype, int n, int cin, int cout, int h, int wd, int act, float alpha, float gain, float clamp,
                          void* workspace, int64_t workspace_bytes, void* stream);
int64_t lvg_sres_dblock_conv1_backward_workspace(int dtype, int n, int cin, int cout, int h, int wd);
int lvg_sres_dblock_conv1_backward(const void* x, const float* fx, const float* fy, int flip, const void* dy, const void* w,
                                   void* dhf, void* dw, int dtype, int n, int cin, int cout, int h, int wd, void* workspace,
                                   int64_t workspace_bytes, void* stream);
int64_t lvg_sres_dblock_fir_adjoint_act_workspace(int dtype, int n, int c, int h, int w);
int lvg_sres_dblock_fir_adjoint_act(const void* dhf, const void* h0, const float* fx, const float* fy, int flip, void* dz,
                                    float* db, void* workspace, int64_t workspace_bytes, int dtype, int n, int c, int h, int w,
                                    int act, float alpha, float gain, float clamp, void* stream);
int64_t lvg_sres_dblock_skip_workspace(int dtype, int n, int cin, int cout, int64_t P);
int lvg_sres_dblock_skip(const void* x, const void* w, const void* r, void* y, int dtype, int n, int cin, int cout, int64_t P,
                         float rscale, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Post-processing of an all-reduced flat gradient buffer, in place and in one pass:
 *   g = g * scale;  NaN -> 0, +inf -> +limit, -inf -> -limit  (finite values untouched)
 * -- the `/ world_size * gain` + `nan_to_num(nan=0, posinf=1e5, neginf=-1e5)` tail of
 * utils.sync_grads (utils.py:116-124) without its extra passes over the buffer. fp32 only.
 */
int lvg_grad_postprocess(float* g, int64_t n, float scale, float limit, void* stream);

/*
 * Fused tail of a training update over flat fp32 buffers (SURVEY.md 8f N3), one pass, in place:
 *   g' = nan_to_num(g * grad_scale, nan = 0, +-inf = +-grad_limit)      only if grad_limit > 0 (utils.py:120-121)
 *   m  = lerp(m, g', 1 - beta1);  v = v * beta2 + (1 - beta2) * g'^2
 *   p  = p - lr / (1 - beta1^step) * m / (sqrt(v) / sqrt(1 - beta2^step) + eps)
 *        -- torch.optim.Adam.step() as the reference configures it (model/video_gan_lres.py:84-85: no weight decay,
 *           no amsgrad), `step` counting from 1
 *   p_ema = lerp(p_ema, p, 1 - ema_beta)                                 only if p_ema != NULL
 *        -- update_G_ema (model/video_gan_lres.py:208-214)
 * write_grad != 0 stores g' back (what utils.sync_grads leaves in .grad). Replaces ~300 per-tensor launches.
 */
int lvg_adam_step(float* p, float* g, float* m, float* v, float* p_ema, int64_t n, float lr, float beta1, float beta2,
                  float eps, int64_t step, float grad_scale, float grad_limit, int write_grad, float ema_beta, void* stream);

/* a = torch.lerp(a, b, weight) over flat fp32 buffers (the buffers of update_G_ema) */
int lvg_lerp(float* a, const float* b, int64_t n, float weight, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LVG_OPS_H_ */
