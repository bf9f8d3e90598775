// fc_tc.cu — the pose-regression head of vgg16_convs on own kernels: RoiPool x2 + add -> fc6 -> fc7 -> fc8 -> tanh
// (lib/networks/vgg16_convs.py:177-197; Network.fc, lib/networks/network.py:392-422: flatten NHWC [N,7,7,512] ->
// 25088 in (h, w, c) order, x @ W[in, out] + b, ReLU; tanh after fc8, network.py:436-438).
//
// At inference the head sees at most 128 ROI rows (MAX_ROI, hough_voting_gpu_op.cu.cc:14), so every layer is a
// 128-row GEMM whose cost is streaming its weights once (fc6: 25088 x 4096 fp16 = 205 MB): HBM-bound.
// Operands are FP16, not BF16 like the trunk: K = 25088 products of 8-bit-mantissa operands leave ~5e-3 relative error on the
// fc6 outputs (measured), 11-bit mantissas ~1e-3 — what the 1e-3 tolerance on the regressed quaternions needs (SURVEY.md
// §8(c)); post-ReLU activations and Kaiming / trained weights sit well inside the fp16 range, and values saturate at 65504.
//   k_roi_pool_pair   ONE kernel pools conv5_3 (scale 1/16) and conv4_3 (scale 1/8) with the RoiPool rule of
//                     roi_pooling_op_gpu.cu.cc:19-101, adds them in fp32 (`pool_score`, vgg16_convs.py:183) and writes the
//                     fp16 A operand [N, 25088] of fc6 directly (no fp32 pooled tensors, no argmax: inference only).
//   k_fc_tc           D[128 rows, BN] partial = A[128, Kslice] * W[BN, Kslice]^T on wgmma (FP16 x FP16 -> FP32 in registers),
//                     both operands K-major, TMA-fed through a 6-stage mbarrier ring; split-K over the grid so that
//                     128 CTAs stream disjoint slices of the weight matrix; partials land in a small fp32 workspace.
//   k_fc_finish       fixed-order sum of the split-K partials + bias + ReLU / tanh -> fp16 activation of the next layer
//                     (or the fp32 `poses_tanh`): run-to-run deterministic.
#include <cuda_fp16.h>
#include <float.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace pcnn {
namespace fctc {

using namespace pcnn::convtc;

constexpr int kFcBN = 128;                        // N tile
constexpr int kFcStages = 6;
constexpr int kFcABytes = kTileM * kKC * 2;       // 16 KB
constexpr int kFcBBytes = kFcBN * kKC * 2;        // 16 KB
constexpr int kFcStage = kFcABytes + kFcBBytes;
constexpr int kFcBarOff = kFcStages * kFcStage;
constexpr int kFcSmem = kFcBarOff + 256 + 1024;
constexpr int kFcThreads = 288;                   // warps 0-7: two consumer warpgroups (rows 0-63 / 64-127), warp 8 TMA producer

// grid = (N / 128, splits, M tiles).  partial: [splits][M][N] f32.
__global__ void __launch_bounds__(kFcThreads, 1)
k_fc_tc(const __grid_constant__ CUtensorMap map_a /*[M][K] f16, box {64, 128}*/,
        const __grid_constant__ CUtensorMap map_w /*[N][K] f16, box {64, 128}*/, float* __restrict__ partial, int M, int N,
        int kchunks_total, int chunks_per_split)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kFcBarOff);
    uint64_t* empty = full + kFcStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * kFcBN, split = blockIdx.y, m0 = blockIdx.z * kTileM;
    const int c_lo = split * chunks_per_split;
    const int c_hi = min(c_lo + chunks_per_split, kchunks_total);
    const int nchunks = c_hi - c_lo;               // >= 1 by construction of the grid

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        for (int s = 0; s < kFcStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int c = 0; c < nchunks; c++) {
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * kFcStage;
                mbar_arrive_expect_tx(&full[stage], kFcStage);
                tma_load_2d(sa, &map_a, &full[stage], (c_lo + c) * kKC, m0);
                tma_load_2d(sa + kFcABytes, &map_w, &full[stage], (c_lo + c) * kKC, n0);
                if (++stage == kFcStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        const int wg = warp >> 2, wq = warp & 3;
        float acc[kFcBN / 2];
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int c = 0; c < nchunks; c++) {
            mbar_wait(&full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * kFcStage);
            const uint64_t da = make_desc(sa + wg * 64 * 128), db = make_desc(sa + kFcABytes);
            acc_fence<kFcBN / 2>(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kKC / 16; k++) wgmma<kFcBN, 1, 0, 0>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (c | k) != 0);
            wgmma_commit();
            acc_fence<kFcBN / 2>(acc);
            if (prev >= 0) {
                wgmma_wait<1>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            prev = stage;
            if (++stage == kFcStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        acc_fence<kFcBN / 2>(acc);
        // epilogue straight from the accumulator fragment: rows (r, r + 8), columns 8 j + 2 (lane % 4) (+ 1)
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int row = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
            if (row < M) {
                float* dst = partial + ((size_t)split * M + row) * N + n0 + 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < kFcBN / 8; j++) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
            }
        }
    }
}

// out[m][n] = act(bias[n] + sum_s partial[s][m][n]) for n < n_valid; act: 0 none, 1 ReLU, 2 tanh.
// out_f16 (row stride ld_out, the next layer's A operand) and / or out_f32 (row stride n_valid).
__global__ void __launch_bounds__(256)
k_fc_finish(const float* __restrict__ partial, int splits, int M, int N, int n_valid, const float* __restrict__ bias, int act,
            __half* __restrict__ out_f16, int ld_out, float* __restrict__ out_f32, const __half* __restrict__ relu_mask /*[M, ld_out] or null*/)
{
    const int nq = N / 4;
    const size_t total = (size_t)M * nq;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int m = (int)(idx / nq), n = (int)(idx % nq) * 4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float4* pp = reinterpret_cast<const float4*>(partial + (size_t)m * N + n);
        const size_t sstride = (size_t)M * N / 4;
        int s = 0;
        for (; s + 4 <= splits; s += 4) {                 // four loads in flight, summed in split order
            const float4 v0 = __ldg(pp + (size_t)s * sstride), v1 = __ldg(pp + (size_t)(s + 1) * sstride);
            const float4 v2 = __ldg(pp + (size_t)(s + 2) * sstride), v3 = __ldg(pp + (size_t)(s + 3) * sstride);
            acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
            acc.x += v1.x; acc.y += v1.y; acc.z += v1.z; acc.w += v1.w;
            acc.x += v2.x; acc.y += v2.y; acc.z += v2.z; acc.w += v2.w;
            acc.x += v3.x; acc.y += v3.y; acc.z += v3.z; acc.w += v3.w;
        }
        for (; s < splits; s++) {
            const float4 v = __ldg(pp + (size_t)s * sstride);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        float o[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (n + j >= n_valid) { o[j] = 0.f; continue; }
            float v = o[j] + (bias ? __ldg(bias + n + j) : 0.f);
            if (act == 1) v = fmaxf(v, 0.f);
            else if (act == 2) v = tanhf(v);
            if (relu_mask && !(__half2float(relu_mask[(size_t)m * ld_out + n + j]) > 0.f)) v = 0.f;   // backward through a ReLU layer
            o[j] = v;
        }
        if (out_f16) {
            __half2 lo = __floats2half2_rn(sat_f16(o[0]), sat_f16(o[1])), hi = __floats2half2_rn(sat_f16(o[2]), sat_f16(o[3]));
            uint2 pk = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
            if (n < ld_out) *reinterpret_cast<uint2*>(out_f16 + (size_t)m * ld_out + n) = pk;
        }
        if (out_f32) {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (n + j < n_valid) out_f32[(size_t)m * n_valid + n + j] = o[j];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// k_roi_pool_pair: out[n, (ph*7+pw)*C + c] = bf16( roipool(f5, 1/16)[n,ph,pw,c] + roipool(f4, 1/8)[n,ph,pw,c] )
// One CTA per (ROI, bin); thread = 8-channel group x row slice of the bin (merged through shared memory).
// Bin arithmetic: roi_pooling_op_gpu.cu.cc:36-62 (round() half away from zero, bin = floor / ceil of ph * bin_size,
// clipped to the map; empty bin -> 0); max from -FLT_MAX with strict `>` — the value is order independent.
// ---------------------------------------------------------------------------------------------
struct RoiBin { int hs, he, ws, we; };

__device__ __forceinline__ RoiBin roi_bin(const float* roi, float scale, int H, int W, int ph, int pw, int PH, int PW)
{
    const int rs_w = (int)roundf(__fmul_rn(roi[2], scale)), rs_h = (int)roundf(__fmul_rn(roi[3], scale));
    const int re_w = (int)roundf(__fmul_rn(roi[4], scale)), re_h = (int)roundf(__fmul_rn(roi[5], scale));
    const int rw = max(re_w - rs_w + 1, 1), rh = max(re_h - rs_h + 1, 1);
    const float bh = __fdiv_rn((float)rh, (float)PH), bw = __fdiv_rn((float)rw, (float)PW);
    RoiBin b;
    b.hs = min(max((int)floorf(__fmul_rn((float)ph, bh)) + rs_h, 0), H);
    b.he = min(max((int)ceilf(__fmul_rn((float)(ph + 1), bh)) + rs_h, 0), H);
    b.ws = min(max((int)floorf(__fmul_rn((float)pw, bw)) + rs_w, 0), W);
    b.we = min(max((int)ceilf(__fmul_rn((float)(pw + 1), bw)) + rs_w, 0), W);
    return b;
}

constexpr int kRpSlices = 4;   // threads that share one (bin, 8-channel group): the bin's rows are dealt round-robin

// running max of rows hs + slice, hs + slice + kRpSlices, ... of a bin, 8 channels; -FLT_MAX where nothing was seen
__device__ __forceinline__ void bin_max8(const __nv_bfloat16* __restrict__ f, int W, int C, const RoiBin& b, int c0, int slice,
                                         float* mx)
{
#pragma unroll
    for (int j = 0; j < 8; j++) mx[j] = -FLT_MAX;
    for (int h = b.hs + slice; h < b.he; h += kRpSlices) {
        const __nv_bfloat16* row = f + ((size_t)h * W) * C + c0;
#pragma unroll 4
        for (int w = b.ws; w < b.we; w++) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(row + (size_t)w * C));
            const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const float2 x = __bfloat1622float2(p[j]);
                mx[2 * j] = fmaxf(mx[2 * j], x.x);
                mx[2 * j + 1] = fmaxf(mx[2 * j + 1], x.y);
            }
        }
    }
}

// grid = (ROI, ph * PW + pw); block = (C / 8 channel groups) x kRpSlices
__global__ void __launch_bounds__(256)
k_roi_pool_pair(const __nv_bfloat16* __restrict__ f5, int H5, int W5, const __nv_bfloat16* __restrict__ f4, int H4, int W4,
                int C, int B, int batch_offset, const float* __restrict__ rois, int roi_stride, int PH, int PW, float scale5,
                float scale4, __half* __restrict__ out)
{
    extern __shared__ float sred[];   // [kRpSlices - 1][groups][16]
    const int n = blockIdx.x, ph = blockIdx.y / PW, pw = blockIdx.y % PW;
    const float* roi = rois + (size_t)n * roi_stride;
    const int b = (int)roi[0] - batch_offset;
    const bool bad = b < 0 || b >= B;          // like the RoiPool kernels: an ROI of another shard pools nothing
    const int groups = C / 8;
    const int g = threadIdx.x % groups, slice = threadIdx.x / groups;
    const int c0 = g * 8;
    const RoiBin b5 = roi_bin(roi, scale5, H5, W5, ph, pw, PH, PW);
    const RoiBin b4 = roi_bin(roi, scale4, H4, W4, ph, pw, PH, PW);
    float m[16];
    if (!bad) {
        bin_max8(f5 + (size_t)b * H5 * W5 * C, W5, C, b5, c0, slice, m);
        bin_max8(f4 + (size_t)b * H4 * W4 * C, W4, C, b4, c0, slice, m + 8);
    }
    if (slice > 0 && !bad) {
        float4* d = reinterpret_cast<float4*>(sred + ((size_t)(slice - 1) * groups + g) * 16);
#pragma unroll
        for (int j = 0; j < 4; j++) d[j] = make_float4(m[4 * j], m[4 * j + 1], m[4 * j + 2], m[4 * j + 3]);
    }
    __syncthreads();
    if (slice != 0) return;
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (!bad) {
        for (int s = 1; s < kRpSlices; s++) {
            const float* q = sred + ((size_t)(s - 1) * groups + g) * 16;
#pragma unroll
            for (int j = 0; j < 16; j++) m[j] = fmaxf(m[j], q[j]);
        }
        const bool e5 = b5.he <= b5.hs || b5.we <= b5.ws, e4 = b4.he <= b4.hs || b4.we <= b4.ws;   // empty bin -> 0 (.cu.cc:64-65)
        __half2* po = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const float a0 = e5 ? 0.f : m[2 * j], a1 = e5 ? 0.f : m[2 * j + 1];
            const float c0v = e4 ? 0.f : m[8 + 2 * j], c1v = e4 ? 0.f : m[8 + 2 * j + 1];
            po[j] = __floats2half2_rn(sat_f16(a0 + c0v), sat_f16(a1 + c1v));
        }
    }
    *reinterpret_cast<uint4*>(out + ((size_t)n * PH * PW + (size_t)ph * PW + pw) * C + c0) = o;
}

}  // namespace fctc
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::fctc;

// split-K plan: as many splits as give ~one wave of CTAs, each with an integer number of 64-element K chunks
static void fc_plan(int M, int N, int K, int* splits, int* chunks_per_split)
{
    const int kchunks = K / kKC, ntiles = N / kFcBN, mtiles = (M + kTileM - 1) / kTileM;
    int want = kNumSMs / (ntiles * mtiles);
    if (want < 1) want = 1;
    if (want > kchunks) want = kchunks;
    if (want > 16) want = 16;              // beyond 16 splits the fixed-order reduction costs more than the streaming gains (fc8)
    int cps = (kchunks + want - 1) / want;
    *chunks_per_split = cps;
    *splits = (kchunks + cps - 1) / cps;
}

extern "C" int pcnn_fc_workspace_bytes(int M, int N, int K, size_t* bytes)
{
    PCNN_REQUIRE(bytes && M >= 1 && N >= kFcBN && N % kFcBN == 0 && K >= kKC && K % kKC == 0,
                 "fc: need M >= 1, N %% 128 == 0, K %% 64 == 0 (got %d, %d, %d)", M, N, K);
    int splits, cps;
    fc_plan(M, N, K, &splits, &cps);
    *bytes = align_up(sizeof(float) * (size_t)splits * M * N, 256);
    return PCNN_OK;
}

// out = act(A[M,K] @ W[N,K]^T + bias): A, W fp16 row-major (K contiguous); bias [n_valid] f32; act 0 none / 1 ReLU / 2 tanh;
// out_f16 [M, ld_out] (optional) and / or out_f32 [M, n_valid] (optional).  Columns n_valid..N of W are padding (zero rows).
static int fc_impl(const void* a_f16, const void* w_f16, const float* bias, int M, int N, int K, int n_valid, int act, void* out_f16,
                   int ld_out, float* out_f32, const void* relu_mask_f16, void* workspace, size_t workspace_bytes, void* stream);

extern "C" int pcnn_fc_f16_tc(const void* a_f16, const void* w_f16, const float* bias, int M, int N, int K, int n_valid,
                              int act, void* out_f16, int ld_out, float* out_f32, void* workspace, size_t workspace_bytes,
                               void* stream)
{
    return fc_impl(a_f16, w_f16, bias, M, N, K, n_valid, act, out_f16, ld_out, out_f32, nullptr, workspace, workspace_bytes, stream);
}

// input-gradient GEMM of a fully connected layer: out = (A @ W^T)[m][n] * [relu_mask[m][n] > 0] (mask = the stored output of the
// ReLU layer below, [M, ld_out] fp16; NULL = no mask), bias NULL allowed
extern "C" int pcnn_fc_dgrad_f16_tc(const void* dy_f16, const void* w_in_out_f16, int M, int N, int K, const void* relu_mask_f16,
                                    void* out_f16, int ld_out, void* workspace, size_t workspace_bytes, void* stream)
{
    return fc_impl(dy_f16, w_in_out_f16, nullptr, M, N, K, N, 0, out_f16, ld_out, nullptr, relu_mask_f16, workspace, workspace_bytes, stream);
}

static int fc_impl(const void* a_f16, const void* w_f16, const float* bias, int M, int N, int K, int n_valid, int act, void* out_f16,
                   int ld_out, float* out_f32, const void* relu_mask_f16, void* workspace, size_t workspace_bytes, void* stream)
{
    PCNN_REQUIRE(a_f16 && w_f16 && workspace && (out_f16 || out_f32), "fc: NULL tensor pointer");
    size_t need = 0;
    int rc = pcnn_fc_workspace_bytes(M, N, K, &need);
    if (rc) return rc;
    PCNN_REQUIRE(n_valid >= 1 && n_valid <= N && act >= 0 && act <= 2, "fc: bad n_valid / act (%d, %d)", n_valid, act);
    PCNN_REQUIRE(!out_f16 || (ld_out % 4 == 0 && ld_out >= 4), "fc: ld_out must be a multiple of 4 (got %d)", ld_out);
    if (workspace_bytes < need) { set_error("fc: workspace too small (%zu < %zu)", workspace_bytes, need); return PCNN_E_WORKSPACE; }
    int splits, cps;
    fc_plan(M, N, K, &splits, &cps);
    CUtensorMap ma, mw;
    rc = make_map_weights(&ma, a_f16, K, M, kTileM, CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
    if (rc) return rc;
    rc = make_map_weights(&mw, w_f16, K, N, kFcBN, CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
    if (rc) return rc;
    PCNN_SMEM_OPTIN(k_fc_tc, kFcSmem, "fc_tc");
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(N / kFcBN, splits, (M + kTileM - 1) / kTileM);
    k_fc_tc<<<grid, kFcThreads, kFcSmem, st>>>(ma, mw, (float*)workspace, M, N, K / kKC, cps);
    rc = check_launch("fc_tc");
    if (rc) return rc;
    const size_t total = (size_t)M * (N / 4);
    int blocks = (int)((total + 255) / 256);
    if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
    k_fc_finish<<<blocks, 256, 0, st>>>((const float*)workspace, splits, M, N, n_valid, bias, act, (__half*)out_f16, ld_out,
                                        out_f32, (const __half*)relu_mask_f16);
    return check_launch("fc_finish");
}

// pool_score = RoiPool(conv5_3, 1/16) + RoiPool(conv4_3, 1/8) (vgg16_convs.py:177-183) flattened to the fc6 operand:
// f5 [B,H5,W5,C] bf16, f4 [B,H4,W4,C] bf16, rois [N, roi_stride] (batch index = rois[:,0] - batch_offset) -> out [N, PH*PW*C] fp16
extern "C" int pcnn_roi_pool_pair_f16(const void* f5, int H5, int W5, const void* f4, int H4, int W4, int C, int B,
                                       int batch_offset, const float* rois, int num_rois, int roi_stride, int pooled_h,
                                       int pooled_w, float scale5, float scale4, void* out_f16, void* stream)
{
    PCNN_REQUIRE(f5 && f4 && rois && out_f16, "roi_pool_pair: NULL tensor pointer");
    PCNN_REQUIRE(C % 8 == 0 && C >= 8 && num_rois >= 1 && roi_stride >= 6 && pooled_h >= 1 && pooled_w >= 1 && B >= 1,
                 "roi_pool_pair: bad shape (C = %d, rois = %d x %d)", C, num_rois, roi_stride);
    PCNN_REQUIRE(pooled_h * pooled_w <= 65535 && C / 8 * kRpSlices <= 256 && 256 % (C / 8) == 0,
                 "roi_pool_pair: needs C / 8 to divide 256 / %d (C = %d)", kRpSlices, C);
    dim3 grid(num_rois, pooled_h * pooled_w);
    const int threads = C / 8 * kRpSlices;
    const size_t smem = sizeof(float) * (size_t)(kRpSlices - 1) * (C / 8) * 16;
    k_roi_pool_pair<<<grid, threads, smem, (cudaStream_t)stream>>>((const __nv_bfloat16*)f5, H5, W5, (const __nv_bfloat16*)f4, H4, W4,
                                                                 C, B, batch_offset, rois, roi_stride, pooled_h, pooled_w, scale5,
                                                                 scale4, (__half*)out_f16);
    return check_launch("roi_pool_pair");
}
