// Pointwise (1x1x1) convolutions on Hopper tensor cores (wgmma), fed straight from the NC(T)HW tensors.
//
// In NC(T)HW a 1x1x1 convolution is one plain GEMM per sample, Y[n] = W X[n]: M = output channels, K = input channels,
// N = the P = T*H*W pixels, contiguous in memory. These layers (skip connections, to/from RGB of the low-res networks) are
// HBM-bound by a wide margin (at most 64 multiply-adds per byte moved), so the kernel is built around moving each tensor
// once: it reads x through a 3-D TMA tensor map [n][channel][pixel] and writes y straight from the accumulators -- no
// re-tiling pass (conv_pack_act_kernel), no halo, no 256-column tile geometry.
//   forward         y[n][co][p] = sum_ci W[co][ci] x[n][ci][p]          (M = cout, K = cin)
//   input gradient  the same kernel on dy with the transposed weight view (M = cin, K = cout)
//
// Products. fp32 tensors are split into bf16 hi + lo halves and every 16-channel k step issues hi*hi, hi*lo, lo*hi (A, B),
// in channel order, into an fp32 accumulator; fp16 tensors issue one fp16 product per k step. That is exactly the product
// sequence conv_igemm_kernel issues for a 1x1x1 layer, and a wgmma result element depends only on its row of A and column
// of B, so the outputs are bit-identical to the engine's whatever the tiling.
//
// Tile = 128 pixels of one sample x one m-tile (128 output channels, or 64 when the GEMM has at most 64 rows). Stage =
// two k steps: the TMA box [1][32 channels][128 pixels] (the 3-D map zero-fills channels past the sample's last one and
// pixels past P, so a partial chunk never reads the next sample) and the packed weight images of the two steps (one bulk
// copy). Roles (384 threads): warp 0 = TMA producer (one lane); warpgroups 1-2 = consumers. The consumers first convert
// the stage's fp32 (fp16) rows into bf16 hi / lo (fp16) B images in the MN-major canonical wgmma layout (pixels are the N
// axis), meet at a named barrier, then issue the products; warpgroup 1 owns accumulator rows 0-63, warpgroup 2 rows
// 64-127 (64-row mode: both read the same 64 rows, each takes 64 of the 128 pixels). The kernel is persistent and the
// stage ring runs across tiles, so the producer streams the next tile while the consumers store this one.
// Weights are split (fp32) and laid out once per call (conv_pw_tc_pack_w_kernel); they are tiny next to the activations.
//
// Envelope: kt = kh = kw = 1, stride 1, no padding, groups 1, no bias / activation epilogue, a 16-byte pixel-row pitch
// (P % 4 == 0 for fp32, P % 8 == 0 for fp16) and 16-byte aligned tensors. conv_igemm.cu routes every such call here
// except the few-channel fp32 ones the streaming SIMT kernels take (conv_pointwise.cu); LVG_CONV_PW_TC=0 sends them to
// the engine instead (A/B comparisons in one process).
#include <cuda.h>
#include <stdlib.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace lvg {
namespace {

using namespace tc;

constexpr int kPtThreads = 384;
constexpr int kPtNP = 128;                       // pixels per tile
constexpr int kPtKS = 2;                         // 16-channel k steps per stage
constexpr int kPtStages = 4;
constexpr int kPtSBO = 272;                      // bytes between 8-pixel groups of a B image: 256 + 16, so that the conversion's
                                                 // stores of consecutive pixel groups fall on different banks
constexpr int kPtBImg = (kPtNP / 8) * kPtSBO;    // one converted 16-channel x 128-pixel B image: 4352 bytes

struct PwTcParams {
    const unsigned char* wp;     // packed weights [mt][kc][nimg][a_img]
    void* y;
    int cout, mt, kc, nimg, a_img, m64;
    int64_t P;
    int ptiles;
    int64_t total_tiles;         // n * ptiles * mt
    int raw_bytes;               // TMA payload of a stage: 32 channels x 128 pixels
    int w_step;                  // bytes of the weight images of one k step: nimg * a_img
    int w_off, b_off, stage_bytes;
};

__device__ __forceinline__ unsigned short pt_bf16_bits(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float pt_bf16_val(unsigned short b) { return __uint_as_float((uint32_t)b << 16); }

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// weights -> K-major images, one per (m-tile, k step, half): element (m, k) of the logical A matrix is w[m * sm + k * sk]
// (forward: sm = cin, sk = 1; input gradient: sm = 1, sk = cin). Image layout as conv_pack_w_kernel's (no swizzle):
// byte offset(m, k) = (k / 8) * (a_img / 2) + m * 16 + (k % 8) * 2, row m = channel m of the m-tile. Rows and channels
// past the matrix are zero. One thread = 8 consecutive k of one row.
template <class TW, bool SPLIT>
__global__ void __launch_bounds__(256) conv_pw_tc_pack_w_kernel(const TW* __restrict__ w, unsigned char* __restrict__ wp, int m_total, int k_total,
                                                                 int64_t sm, int64_t sk, int mt, int kc, int rows)
{
    constexpr int NIMG = SPLIT ? 2 : 1;
    const int img = rows * 32;
    const int total = mt * kc * 2 * rows;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int r = i % rows;
        const int k8 = (i / rows) % 2;
        const int kci = (i / (2 * rows)) % kc;
        const int mti = i / (2 * rows * kc);
        const int m = mti * rows + r;
        alignas(16) unsigned short v[8], vlo[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int k = kci * 16 + k8 * 8 + j;
            const bool ok = m < m_total && k < k_total;
            if constexpr (SPLIT) {
                const float f = ok ? __ldg(reinterpret_cast<const float*>(w) + m * sm + k * sk) : 0.f;
                v[j] = pt_bf16_bits(f);
                vlo[j] = pt_bf16_bits(f - pt_bf16_val(v[j]));
            } else {
                v[j] = ok ? __half_as_ushort(__ldg(reinterpret_cast<const __half*>(w) + m * sm + k * sk)) : (unsigned short)0;
            }
        }
        unsigned char* d = wp + ((int64_t)(mti * kc + kci) * NIMG) * img + k8 * (img / 2) + r * 16;
        *reinterpret_cast<uint4*>(d) = *reinterpret_cast<const uint4*>(v);
        if constexpr (SPLIT) *reinterpret_cast<uint4*>(d + img) = *reinterpret_cast<const uint4*>(vlo);
    }
}

// Stage layout: [raw: 32 channels x 128 pixels as TMA wrote them][weight images of the k steps][converted B images:
// per k step nimg images of kPtBImg bytes]. B image (MN-major, no swizzle): byte offset(k, px) = (px / 8) * kPtSBO +
// (k / 8) * 128 + (k % 8) * 16 + (px % 8) * 2 -- 8 x 8 core matrices, LBO = 128 (next 8 channels), SBO = kPtSBO.
// NW: MMA width of a consumer (128; 64 in 64-row mode).
template <bool BF16, int NW>
__global__ void __launch_bounds__(kPtThreads, 1) conv_pw_tc_kernel(const __grid_constant__ CUtensorMap tmx, const PwTcParams p)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full_bar[kPtStages], empty_bar[kPtStages];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);

    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);
    const int kchunks = (p.kc + kPtKS - 1) / kPtKS;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kPtStages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        if (warp == 0 && elect_one()) {
            int it = 0;
            for (int64_t L = blockIdx.x; L < p.total_tiles; L += gridDim.x) {
                // m-tile fastest: CTAs running side by side share one x tile in L2
                const int mti = (int)(L % p.mt);
                const int64_t r = L / p.mt;
                const int pt = (int)(r % p.ptiles);
                const int n = (int)(r / p.ptiles);
                const unsigned char* wpm = p.wp + (int64_t)mti * p.kc * p.w_step;
                for (int kcix = 0; kcix < kchunks; kcix++, it++) {
                    const int s = it % kPtStages;
                    if (it >= kPtStages) mbar_wait(&empty_bar[s], (uint32_t)((it / kPtStages - 1) & 1));
                    unsigned char* st = smem + (size_t)s * p.stage_bytes;
                    const int k0 = kcix * kPtKS;
                    const int nks = min(kPtKS, p.kc - k0);
                    const uint32_t wb = (uint32_t)(nks * p.w_step);
                    mbar_expect_tx(&full_bar[s], wb + (uint32_t)p.raw_bytes);
                    bulk_copy_g2s(st + p.w_off, wpm + (int64_t)k0 * p.w_step, wb, &full_bar[s]);
                    tma_load_3d(st, &tmx, pt * kPtNP, k0 * 16, n, &full_bar[s]);
                }
            }
        }
    } else {
        const int cw = wg - 1;
        const int ctid = threadIdx.x - 128;              // 0..255: both consumer warpgroups convert
        const int tid = threadIdx.x % 128, wq = tid / 32;
        const uint32_t a_hi = desc_hi(128), b_hi = desc_hi(kPtSBO);
        const uint32_t a_lo_img = (uint32_t)p.a_img >> 4, b_lo_img = (uint32_t)kPtBImg >> 4;
        const uint32_t a_row0 = p.m64 ? 0u : (uint32_t)cw * 1024u;      // this warpgroup's 64 rows of a 128-row image
        const int col0 = p.m64 ? cw * NW : 0;                            // 64-row mode: this warpgroup's pixels
        int it = 0;
        for (int64_t L = blockIdx.x; L < p.total_tiles; L += gridDim.x) {
            const int mti = (int)(L % p.mt);
            const int64_t r = L / p.mt;
            const int pt = (int)(r % p.ptiles);
            const int n = (int)(r / p.ptiles);
            float acc[NW / 2];
#pragma unroll
            for (int i = 0; i < NW / 2; i++) acc[i] = 0.f;
            int prev = -1;
            for (int kcix = 0; kcix < kchunks; kcix++, it++) {
                const int s = it % kPtStages;
                const int nks = min(kPtKS, p.kc - kcix * kPtKS);
                unsigned char* st = smem + (size_t)s * p.stage_bytes;
                unsigned char* bimg = st + p.b_off;
                mbar_wait(&full_bar[s], (uint32_t)((it / kPtStages) & 1));
                // ---- raw rows -> B images (the slot's B images were last read by MMAs that completed before it was refilled)
                if constexpr (BF16) {
                    const float* raw = reinterpret_cast<const float*>(st);
                    for (int i = ctid; i < nks * 16 * (kPtNP / 4); i += 256) {
                        const int q = i % (kPtNP / 4), k = i / (kPtNP / 4);
                        const float4 v = *reinterpret_cast<const float4*>(raw + k * kPtNP + 4 * q);
                        const float f[4] = {v.x, v.y, v.z, v.w};
                        alignas(8) unsigned short hi[4], lo[4];
#pragma unroll
                        for (int e = 0; e < 4; e++) {
                            hi[e] = pt_bf16_bits(f[e]);
                            lo[e] = pt_bf16_bits(f[e] - pt_bf16_val(hi[e]));
                        }
                        const int j = k / 16, kk = k % 16;
                        unsigned char* d = bimg + j * (2 * kPtBImg) + (q / 2) * kPtSBO + (kk / 8) * 128 + (kk % 8) * 16 + (q % 2) * 8;
                        *reinterpret_cast<uint2*>(d) = *reinterpret_cast<const uint2*>(hi);
                        *reinterpret_cast<uint2*>(d + kPtBImg) = *reinterpret_cast<const uint2*>(lo);
                    }
                } else {
                    const uint4* raw = reinterpret_cast<const uint4*>(st);
                    for (int i = ctid; i < nks * 16 * (kPtNP / 8); i += 256) {
                        const int g = i % (kPtNP / 8), k = i / (kPtNP / 8);
                        const int j = k / 16, kk = k % 16;
                        *reinterpret_cast<uint4*>(bimg + j * kPtBImg + g * kPtSBO + (kk / 8) * 128 + (kk % 8) * 16) = raw[k * (kPtNP / 8) + g];
                    }
                }
                fence_proxy_async();                    // generic-proxy stores -> the MMAs' async-proxy reads
                consumer_bar_sync();
                wgmma_fence();
                const uint32_t sa = smem_u32(st + p.w_off), sb = smem_u32(bimg) + (uint32_t)(col0 / 8) * kPtSBO;
                for (int j = 0; j < nks; j++) {
                    const uint32_t a_lo = desc_lo(sa + (uint32_t)(j * p.w_step) + a_row0, (uint32_t)p.a_img / 2);
                    const uint32_t b_lo = desc_lo(sb + (uint32_t)(j * p.nimg * kPtBImg), 128);
                    // fp16: one product; split: hi*hi, hi*lo, lo*hi (A image hi, hi, lo; B image hi, lo, hi) -- conv_igemm_kernel's order
                    wgmma_m64nNk16<BF16, NW, 0, 1>(acc, a_lo, a_hi, b_lo, b_hi);
                    if constexpr (BF16) {
                        wgmma_m64nNk16<BF16, NW, 0, 1>(acc, a_lo, a_hi, b_lo + b_lo_img, b_hi);
                        wgmma_m64nNk16<BF16, NW, 0, 1>(acc, a_lo + a_lo_img, a_hi, b_lo, b_hi);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                        // the group of the previous stage has completed: release its slot
                mbar_arrive_if(&empty_bar[prev >= 0 ? prev : 0], prev >= 0 && tid == 0);
                prev = s;
            }
            wgmma_wait<0>();
            mbar_arrive_if(&empty_bar[prev], tid == 0);

            // ---- epilogue: registers -> y. This thread holds rows 16 wq + lane / 4 (+ 8) and column pairs 8 j + 2 (lane % 4):
            // 8-byte (fp32) / 4-byte (fp16) stores, a warp's store covers 8 channel rows x 32 (16) contiguous bytes
            const int64_t p0 = (int64_t)pt * kPtNP;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row = wq * 16 + lane / 4 + 8 * h;
                const int co = p.m64 ? row : mti * 128 + cw * 64 + row;
                if (co >= p.cout) continue;
                const int64_t base = ((int64_t)n * p.cout + co) * p.P + p0;
#pragma unroll
                for (int j = 0; j < NW / 8; j++) {
                    const int col = col0 + j * 8 + 2 * (lane % 4);
                    if (p0 + col >= p.P) continue;                 // P is even: the pair is whole
                    const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                    if constexpr (BF16) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.y) + base + col) = make_float2(v0, v1);
                    else *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.y) + base + col) = __floats2half2_rn(v0, v1);
                }
            }
        }
    }
}

typedef CUresult (*PtEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PtEncodeFn pt_encode_fn()
{
    static PtEncodeFn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
        return reinterpret_cast<PtEncodeFn>(f);
    }();
    return fn;
}

struct PwTcGeom { int kc, mt, m64, nimg, a_img; int64_t w_bytes; };

PwTcGeom pw_tc_geometry(int split, int ck, int cm)
{
    PwTcGeom g;
    g.kc = (ck + 15) / 16;
    g.m64 = cm <= 64 ? 1 : 0;
    g.mt = g.m64 ? 1 : (cm + 127) / 128;
    g.nimg = split ? 2 : 1;
    g.a_img = g.m64 ? 2048 : 4096;
    g.w_bytes = (int64_t)g.mt * g.kc * g.nimg * g.a_img;
    return g;
}

}  // namespace

// the route: LVG_CONV_PW_TC=0 keeps these calls on the engine (read on every call, so one process can compare both)
bool pw_tc_supported(int dtype, int groups, int cin, int cout, int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride, int64_t P)
{
    const char* e = getenv("LVG_CONV_PW_TC");
    if (e && e[0] == '0') return false;
    const int64_t align = dtype == LVG_F32 ? 4 : 8;
    return (dtype == LVG_F32 || dtype == LVG_F16) && groups == 1 && kt == 1 && kh == 1 && kw == 1 && pad_t == 0 && pad_h == 0 && pad_w == 0 &&
           stride == 1 && cin >= 1 && cout >= 1 && P >= align && P % align == 0 && P / kPtNP < (1ll << 30);
}

// bytes of workspace the call needs (the packed weights): never more than the engine's packed weights of the same GEMM
int64_t pw_tc_workspace(int dtype, int ck, int cm) { return pw_tc_geometry(dtype == LVG_F32, ck, cm).w_bytes + 256; }

// y[n][m][p] = sum_k w[m * w_sm + k * w_sk] * x[n][k][p]: x has ck channels, y cm (forward: ck = cin, cm = cout, w_sm = cin,
// w_sk = 1; input gradient: x = dy, ck = cout, cm = cin, w_sm = 1, w_sk = cin)
int pw_tc_conv(const void* x, const void* w, void* y, int dtype, int n, int ck, int cm, int64_t P, int64_t w_sm, int64_t w_sk, void* workspace,
               int64_t workspace_bytes, cudaStream_t s)
{
    const int split = dtype == LVG_F32 ? 1 : 0;
    const int es = split ? 4 : 2;
    const PwTcGeom g = pw_tc_geometry(split, ck, cm);
    LVG_REQUIRE(aligned16(x) && aligned16(y), "pointwise conv: tensors must be 16-byte aligned");
    LVG_REQUIRE(workspace && aligned16(workspace) && workspace_bytes >= g.w_bytes, "pointwise conv: workspace too small");
    PtEncodeFn enc = pt_encode_fn();
    LVG_REQUIRE(enc != nullptr, "pointwise conv: cuTensorMapEncodeTiled is not available from this driver");

    unsigned char* wp = reinterpret_cast<unsigned char*>(workspace);
    {
        const int rows = g.m64 ? 64 : 128;
        const int total = g.mt * g.kc * 2 * rows;
        const int blocks = (total + 255) / 256;
        if (split) conv_pw_tc_pack_w_kernel<float, true><<<blocks, 256, 0, s>>>((const float*)w, wp, cm, ck, w_sm, w_sk, g.mt, g.kc, rows);
        else conv_pw_tc_pack_w_kernel<__half, false><<<blocks, 256, 0, s>>>((const __half*)w, wp, cm, ck, w_sm, w_sk, g.mt, g.kc, rows);
        LVG_LAUNCH_CHECK();
    }

    // x as [n][ck][P] elements: box [1][32 channels][128 pixels], zero fill past every edge
    CUtensorMap tm;
    {
        const cuuint64_t dims[3] = {(cuuint64_t)P, (cuuint64_t)ck, (cuuint64_t)n};
        const cuuint64_t strides[2] = {(cuuint64_t)P * es, (cuuint64_t)P * ck * es};
        const cuuint32_t box[3] = {(cuuint32_t)kPtNP, (cuuint32_t)(kPtKS * 16), 1};
        const cuuint32_t estr[3] = {1, 1, 1};
        const CUresult r = enc(&tm, split ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(x), dims, strides,
                               box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        LVG_REQUIRE(r == CUDA_SUCCESS, "pointwise conv: cuTensorMapEncodeTiled failed (%d)", (int)r);
    }

    PwTcParams p;
    memset(&p, 0, sizeof(p));
    p.wp = wp; p.y = y;
    p.cout = cm; p.mt = g.mt; p.kc = g.kc; p.nimg = g.nimg; p.a_img = g.a_img; p.m64 = g.m64;
    p.P = P;
    p.ptiles = (int)((P + kPtNP - 1) / kPtNP);
    p.total_tiles = (int64_t)n * p.ptiles * g.mt;
    p.raw_bytes = kPtKS * 16 * kPtNP * es;
    p.w_step = g.nimg * g.a_img;
    p.w_off = p.raw_bytes;
    p.b_off = p.w_off + kPtKS * p.w_step;
    p.stage_bytes = p.b_off + kPtKS * g.nimg * kPtBImg;
    const size_t smem = (size_t)kPtStages * p.stage_bytes + 128;

    void (*kern)(const CUtensorMap, const PwTcParams) =
        split ? (g.m64 ? conv_pw_tc_kernel<true, 64> : conv_pw_tc_kernel<true, 128>) : (g.m64 ? conv_pw_tc_kernel<false, 64> : conv_pw_tc_kernel<false, 128>);
    LVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t ctas = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
    kern<<<(unsigned)ctas, kPtThreads, smem, s>>>(tm, p);
    LVG_LAUNCH_CHECK();
    return LVG_OK;
}

}  // namespace lvg
