// conv_tc.cu — the VGG16 convolution stack on the sm_90a tensor cores (wgmma + TMA + mbarrier).
//
// Behavioural spec: Network.conv, lib/networks/network.py:159-188 (NHWC x HWIO, SAME padding,
// stride 1, bias add, optional ReLU) as wired by lib/networks/vgg16_convs.py:80-97, 128-163.
// The reference runs tf.nn.conv2d -> cuDNN in fp32; here the convolution is an implicit GEMM
//
//      D[m, n] = sum_{tap, c} A_tap[m, c] * Wt[n, tap*Cin + c],      m = pixel of an 8x16 (or 16x16) tile
//
// with BF16 operands and FP32 accumulation (precision is stated with every number, DESIGN.md §4):
//   * im2col is never materialised: for every filter tap the A operand of a tile is ONE 4-D TMA
//     box {64 ch, 16 w, 8 h, 1 n} (256-pixel tile: {64, 16, 16, 1}) of the NHWC activation tensor at the tap's (dy, dx)
//     offset; out-of-image coordinates are zero-filled by the TMA unit = SAME padding;
//   * the box lands in shared memory as 128 (256) rows x 128 B with the 128-byte swizzle, which is
//     exactly the canonical K-major wgmma operand layout, so wgmma reads it in place;
//   * warp roles: warps 0-7 = two consumer warpgroups (pixel rows 0-63 / 64-127 of each 128-pixel half): wgmma with the
//     accumulators in registers, then the epilogue (bias, ReLU, bf16 pack, TMA store) from registers; warpgroup 2
//     (warps 8-11) gives its registers to the consumers (setmaxnreg: 2 x 128 x 232 + 128 x 40 <= 64 K) and one thread of
//     it is the TMA producer, which keeps filling the stage ring during the epilogue.  Persistent CTAs, one per SM,
//     static round-robin tile schedule.
#include <cuda.h>
#include <cuda_bf16.h>

#include <type_traits>

#include "common.cuh"
#include "tc_common.cuh"

namespace pcnn {
namespace convtc {

constexpr int kTileH = 8, kTileW = 16;                            // 128 output pixels per tile (kTileM, tc_common.cuh)
static_assert(kTileH * kTileW == kTileM, "pixel tile = two wgmma M blocks");
constexpr int kABytes = kTileM * kKC * 2;                         // 16 KB
constexpr int kConsumers = 256;                                   // two consumer warpgroups
constexpr int kProducerWarp = kConsumers / 32;                    // warp 8
constexpr int kThreadsConv = kConsumers + 128;                    // k_conv_tc: consumer warpgroups + a producer warpgroup
constexpr int kConsumerRegs = 232, kProducerRegs = 40;            // k_conv_tc after setmaxnreg: 256 x 232 + 128 x 40 <= 64 K
constexpr int kThreadsRow = kConsumers + 32;                      // k_conv_row2: consumer warpgroups + one producer warp (168 regs)
constexpr int kStageBytes = 16 * 1024;                            // epilogue staging: one 64-channel group

struct ConvParams {
    int B, H, W, Cin, Cout;
    int taps, ksize;          // 9 / 3 or 1 / 1
    int tiles_h, tiles_w, n_tiles_n, total_tiles;
    int tile_h, tile_w;       // k_conv_tc: pixel tile (tile_h * tile_w = 128; 8 x 16, or 16 x 8 when that wastes fewer pixels)
    int relu;
    int pool;                 // 1: the epilogue applies the 2x2 / stride-2 max pool and stores ONLY the pooled tensor
    int kc_outer;             // k_conv_tc<BN, 256>: 1 = K steps chunk-outer (ks = c * taps + tap), 0 = tap-outer
    const float* bias;
};

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// a warp of a consumer warpgroup is done with a stage (its wgmma reads of it have completed)
__device__ __forceinline__ void release(uint64_t* bar, int lane)
{
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
}

// 64 channels of the fragment rows (row, row + 8) — the 32 accumulator registers of one 64-column group — plus bias,
// optional ReLU, bf16 -> the swizzled 128-byte staging rows that the TMA store reads (q = lane % 4)
__device__ __forceinline__ void stage_rows(uint8_t* ob, const float* a, const float* bias, int relu, int row, int q)
{
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int r = row + 8 * i;
#pragma unroll
        for (int jj = 0; jj < 8; jj++) {
            const int c = 8 * jj + 2 * q;
            float v0 = a[4 * jj + 2 * i] + __ldg(bias + c), v1 = a[4 * jj + 2 * i + 1] + __ldg(bias + c + 1);
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            *reinterpret_cast<uint32_t*>(ob + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * q) = pack_bf16(v0, v1);
        }
    }
}

// fused max_pool 2x2/2 (network.py:303-310) of a staged 8 x 16 tile (row m = 16 h + w), in place: pooled row
// p = 8 ph + pw is the max of rows 32 ph + 2 pw + {0, 1, 16, 17}.  One 16-byte piece per consumer thread.  max on the
// bf16 values = bf16 of the fp32 max (rounding is monotone).
__device__ __forceinline__ void pool_staged(uint8_t* ob, int t)
{
    const int p = t >> 3, piece = t & 7;
    const int m = 32 * (p >> 3) + 2 * (p & 7);
    const int rows[4] = {m, m + 1, m + 16, m + 17};
    __nv_bfloat162 v[4];
    uint4 x = *reinterpret_cast<const uint4*>(ob + rows[0] * 128 + ((piece ^ (rows[0] & 7)) << 4));
    *reinterpret_cast<uint4*>(v) = x;
#pragma unroll
    for (int k = 1; k < 4; k++) {
        uint4 y = *reinterpret_cast<const uint4*>(ob + rows[k] * 128 + ((piece ^ (rows[k] & 7)) << 4));
        const __nv_bfloat162* yv = reinterpret_cast<const __nv_bfloat162*>(&y);
#pragma unroll
        for (int q = 0; q < 4; q++) v[q] = __hmax2(v[q], yv[q]);
    }
    consumer_sync();   // every source row has been read before any pooled row overwrites one
    *reinterpret_cast<uint4*>(ob + p * 128 + ((piece ^ (p & 7)) << 4)) = *reinterpret_cast<const uint4*>(v);
}

// BM = pixels of a tile: 128 (8 x 16 or 16 x 8), or 256 (16 x 16 = two 8 x 16 halves, rows 0-127 = image rows h0 .. h0 + 7)
template <int BN, int BM>
struct SmemPlan {
    static constexpr int kABytesT = BM * kKC * 2;
    static constexpr int kBBytes = BN * kKC * 2;
    static constexpr int kStage = kABytesT + kBBytes;
    static constexpr int kStages = BN == 256 || BM == 256 ? 4 : (BN == 128 ? 6 : 8);
    static constexpr int kOutBufs = 2;
    static constexpr int kBarOff = kStages * kStage + kOutBufs * kStageBytes;
    static constexpr int kTotal = kBarOff + 256 + 1024;  // barriers + alignment slack
};

// BM = 128: consumer warpgroup g owns the m64 block g; K order tap-outer (ks = tap * kchunks + c).
// BM = 256: warpgroup g owns the m64 blocks g and g + 2 (its rows of both 8 x 16 halves, one accumulator each); K order
// chunk-outer (the order of row mode) or tap-outer as p.kc_outer says (conv_bf16_tc_impl).
template <int BN, int BM>
__global__ void __launch_bounds__(kThreadsConv, 1)
k_conv_tc(const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_w,
          const __grid_constant__ CUtensorMap map_out, const ConvParams p)  // map_out: box {64,16,8,1}, or {64,8,4,1} of the pooled tensor
{
    static_assert(BM == 128 || (BM == 256 && BN <= 128), "k_conv_tc: BM = 256 needs BN <= 128 (accumulator registers)");
    using Plan = SmemPlan<BN, BM>;
    constexpr int kMB = BM / kTileM;                   // accumulators (8 x 16 halves) per consumer thread
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* out_stage = smem + Plan::kStages * Plan::kStage;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Plan::kBarOff);
    uint64_t* empty = full + Plan::kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kchunks = p.Cin / kKC;
    const int ksteps = p.taps * kchunks;

    if (warp == kProducerWarp && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_in) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
        for (int s = 0; s < Plan::kStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumers / 32); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= kProducerWarp) {
        // ===================== TMA producer: one thread of warpgroup 2 =====================
        setmaxnreg_dec<kProducerRegs>();
        if (warp == kProducerWarp && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                const int nt = tile % p.n_tiles_n;
                int rest = tile / p.n_tiles_n;
                const int tw = rest % p.tiles_w; rest /= p.tiles_w;
                const int th = rest % p.tiles_h;
                const int img = rest / p.tiles_h;
                const int h0 = th * p.tile_h, w0 = tw * p.tile_w, n0 = nt * BN;
                const int pad = p.ksize / 2;
#pragma unroll 1   // the producer runs on 40 registers
                for (int ks = 0; ks < ksteps; ks++) {
                    const bool kc_outer = BM == 256 && p.kc_outer;
                    const int tap = kc_outer ? ks % p.taps : ks / kchunks;
                    const int c0 = (kc_outer ? ks / p.taps : ks % kchunks) * kKC;
                    const int dy = tap / p.ksize - pad, dx = tap % p.ksize - pad;
                    mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * Plan::kStage;
                    mbar_arrive_expect_tx(&full[stage], Plan::kStage);
                    tma_load_4d(sa, &map_in, &full[stage], c0, w0 + dx, h0 + dy, img);
                    tma_load_2d(sa + Plan::kABytesT, &map_w, &full[stage], tap * p.Cin + c0, n0);
                    if (++stage == Plan::kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: MMA + epilogue =====================
        setmaxnreg_inc<kConsumerRegs>();
        const int wg = warp >> 2, wq = warp & 3;
        const int row = wg * 64 + wq * 16 + (lane >> 2);   // first of the two rows (pixels) of a 128-pixel half this thread holds
        float acc[kMB][BN / 2];                            // acc[h]: the thread's rows of half h
        int stage = 0, obuf = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
            const int nt = tile % p.n_tiles_n;
            int rest = tile / p.n_tiles_n;
            const int tw = rest % p.tiles_w; rest /= p.tiles_w;
            const int th = rest % p.tiles_h;
            const int img = rest / p.tiles_h;
            const int h0 = th * p.tile_h, w0 = tw * p.tile_w, n0 = nt * BN;
            int prev = -1;
            for (int ks = 0; ks < ksteps; ks++) {
                mbar_wait(&full[stage], phase);
                const uint32_t sa = smem_u32(smem + stage * Plan::kStage);
                const uint64_t db = make_desc(sa + Plan::kABytesT);
#pragma unroll
                for (int h = 0; h < kMB; h++) acc_fence<BN / 2>(acc[h]);
                wgmma_fence();
#pragma unroll
                for (int h = 0; h < kMB; h++) {
                    const uint64_t da = make_desc(sa + (h * 2 + wg) * 64 * 128);   // m64 block wg of half h
#pragma unroll
                    for (int k = 0; k < kKC / 16; k++)
                        wgmma<BN, 0, 0, 0>(acc[h], da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (ks | k) != 0);
                }
                wgmma_commit();
#pragma unroll
                for (int h = 0; h < kMB; h++) acc_fence<BN / 2>(acc[h]);
                if (prev >= 0) {   // the previous stage's MMAs are complete: its slot may be refilled
                    wgmma_wait<1>();
                    release(&empty[prev], lane);
                }
                prev = stage;
                if (++stage == Plan::kStages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int h = 0; h < kMB; h++) acc_fence<BN / 2>(acc[h]);
            release(&empty[prev], lane);
#pragma unroll
            for (int h = 0; h < kMB; h++) {
                // a second half wholly below the image has nothing to store (the condition is uniform over the CTA)
                if (h > 0 && h0 + 8 * h >= p.H) break;
#pragma unroll
                for (int g = 0; g < BN / 64; g++) {
                    // staging buffer obuf must have been read out by the TMA store issued two groups ago
                    if (threadIdx.x == 0) tma_store_wait_read<1>();
                    consumer_sync();
                    uint8_t* ob = out_stage + obuf * kStageBytes;
                    stage_rows(ob, acc[h] + g * 32, p.bias + n0 + g * 64, p.relu, row, lane & 3);
                    if (p.pool) {
                        consumer_sync();
                        pool_staged(ob, threadIdx.x);
                    }
                    fence_proxy_async();
                    consumer_sync();
                    if (threadIdx.x == 0) {   // half h: image rows h0 + 8 h .. h0 + 8 h + 7 (pooled: 4 rows from h0 / 2 + 4 h)
                        if (!p.pool) tma_store_4d(&map_out, ob, n0 + g * 64, w0, h0 + 8 * h, img);
                        else tma_store_4d(&map_out, ob, n0 + g * 64, w0 >> 1, (h0 >> 1) + 4 * h, img);
                        tma_store_commit();
                    }
                    obuf ^= 1;
                }
            }
        }
        if (threadIdx.x == 0) tma_store_wait_all();
    }
}

// ---------------------------------------------------------------------------------------------
// Row mode for the K-small layers (conv1_2, conv2_x: Cin, Cout <= 128), which are bound by L2 -> SM operand
// traffic in the tile kernel (every tap re-fetches its A tile).
// A work item is TWO output rows x 128 pixels of one image:
//   * per 64-channel chunk ONE TMA box {64 ch, 130 px, 4 rows} (halo included) is loaded; the A operand of
//     tap (r, s) for output row j is the 128 consecutive patch rows starting at ((r + j) * 130 + s): a
//     row-shifted view of the same shared-memory patch (the swizzle is a function of the shared-memory address, so
//     a start address that is 128-B but not 1024-B aligned needs no descriptor change);
//   * every weight stage feeds both output rows (two register accumulators), halving the weight traffic as well;
//   * the two rows of a pair are exactly the rows a 2x2 max pool combines, so the pool stays fused: vertical
//     max in registers (the same thread holds the same pixel of both rows), horizontal max by shuffle.
// Operand bytes per 128 output pixels drop from 9 * (16 + BN/8) KB to (32.5 + 4.5 * BN/8) KB per chunk.
// ---------------------------------------------------------------------------------------------
constexpr int kRowPx = 128, kPatchW = 130, kPatchH = 4;
constexpr int kPatchBytes = kPatchW * kPatchH * 128;  // 66,560 = 65 * 1024
constexpr int kRowAStages = 2;

// BN = 64.  RESB (Cin = 64 only): the nine 8-KB weight slices of the CTA's N tile stay resident in shared memory for
// the whole kernel; every CTA keeps one N tile (nt = blockIdx.x % n_tiles_n).  The epilogue staging shrinks to 16 KB
// to make room.
template <int BN, bool RESB>
struct RowPlan {
    static constexpr int kBBytes = BN * 128;
    static constexpr int kBStages = RESB ? 9 : 6;
    static constexpr int kBOff = kRowAStages * kPatchBytes;
    static constexpr int kOutOff = kBOff + kBStages * kBBytes;
    static constexpr int kOutBytes = RESB ? kStageBytes : 2 * kStageBytes;
    static constexpr int kBarOff = kOutOff + kOutBytes;
    static constexpr int kTotal = kBarOff + 256 + 1024;
};

template <int BN, bool RESB>
__global__ void __launch_bounds__(kThreadsRow, 1)
k_conv_row2(const __grid_constant__ CUtensorMap map_in /*box {64,130,4,1}*/, const __grid_constant__ CUtensorMap map_w,
            const __grid_constant__ CUtensorMap map_out /*box {64,128,1,1}, or {64,64,1,1} of the pooled tensor*/,
            const ConvParams p)
{
    using Plan = RowPlan<BN, RESB>;
    static_assert(BN == 64, "row mode: 64-channel N tiles");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sB = smem + Plan::kBOff;
    uint8_t* out_stage = smem + Plan::kOutOff;
    uint64_t* fullA = reinterpret_cast<uint64_t*>(smem + Plan::kBarOff);
    uint64_t* emptyA = fullA + kRowAStages;
    uint64_t* fullB = emptyA + kRowAStages;
    uint64_t* emptyB = fullB + Plan::kBStages;
    uint64_t* wbar = emptyB + Plan::kBStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kchunks = p.Cin / kKC;
    // work items of this CTA: RESB -> fixed N tile, spatial tiles strided; otherwise all (spatial, N) tiles strided
    const int tile0 = RESB ? blockIdx.x / p.n_tiles_n : blockIdx.x;
    const int tstep = RESB ? gridDim.x / p.n_tiles_n : gridDim.x;
    const int tcount = RESB ? p.total_tiles / p.n_tiles_n : p.total_tiles;
    const int nt_fixed = blockIdx.x % p.n_tiles_n;
    // tiles_h = row pairs, tiles_w = 128-pixel segments
    if (warp == kProducerWarp && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_in) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
        for (int s = 0; s < kRowAStages; s++) { mbar_init(&fullA[s], 1); mbar_init(&emptyA[s], kConsumers / 32); }
        for (int s = 0; s < Plan::kBStages; s++) { mbar_init(&fullB[s], 1); mbar_init(&emptyB[s], kConsumers / 32); }
        mbar_init(wbar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            int sa = 0, sb = 0;
            uint32_t pa = 0, pb = 0;
            if (RESB) {
                mbar_arrive_expect_tx(wbar, 9 * Plan::kBBytes);
                for (int tap = 0; tap < 9; tap++)      // resident slices in tap order
                    tma_load_2d(sB + tap * Plan::kBBytes, &map_w, wbar, tap * p.Cin, nt_fixed * BN);
            }
            for (int tile = tile0; tile < tcount; tile += tstep) {
                const int nt = RESB ? nt_fixed : tile % p.n_tiles_n;
                int rest = RESB ? tile : tile / p.n_tiles_n;
                const int tw = rest % p.tiles_w; rest /= p.tiles_w;
                const int yp = rest % p.tiles_h;
                const int img = rest / p.tiles_h;
                const int y0 = 2 * yp, x0 = tw * kRowPx, n0 = nt * BN;
                for (int c = 0; c < kchunks; c++) {
                    mbar_wait(&emptyA[sa], pa ^ 1);
                    mbar_arrive_expect_tx(&fullA[sa], kPatchBytes);
                    tma_load_4d(smem + sa * kPatchBytes, &map_in, &fullA[sa], c * kKC, x0 - 1, y0 - 1, img);
                    if (++sa == kRowAStages) { sa = 0; pa ^= 1; }
                    if (!RESB) {
                        for (int tap = 0; tap < 9; tap++) {
                            mbar_wait(&emptyB[sb], pb ^ 1);
                            mbar_arrive_expect_tx(&fullB[sb], Plan::kBBytes);
                            tma_load_2d(sB + sb * Plan::kBBytes, &map_w, &fullB[sb], tap * p.Cin + c * kKC, n0);
                            if (++sb == Plan::kBStages) { sb = 0; pb ^= 1; }
                        }
                    }
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: thread = pixels (row, row + 8) of both output rows =====================
        constexpr int kH = BN / 2;                  // accumulator registers of one output row (m64nBN): row j at acc[j * kH]
        const int wg = warp >> 2, wq = warp & 3;
        const int row = wg * 64 + wq * 16 + (lane >> 2);
        float acc[2 * kH];
        int sa = 0, sb = 0, obuf = 0;
        uint32_t pa = 0, pb = 0;
        if (RESB) mbar_wait(wbar, 0);
        for (int tile = tile0; tile < tcount; tile += tstep) {
            const int nt = RESB ? nt_fixed : tile % p.n_tiles_n;
            int rest = RESB ? tile : tile / p.n_tiles_n;
            const int tw = rest % p.tiles_w; rest /= p.tiles_w;
            const int yp = rest % p.tiles_h;
            const int img = rest / p.tiles_h;
            const int y0 = 2 * yp, x0 = tw * kRowPx, n0 = nt * BN;
            for (int c = 0; c < kchunks; c++) {
                mbar_wait(&fullA[sa], pa);
                const uint32_t a_base = smem_u32(smem + sa * kPatchBytes) + wg * 64 * 128;
                if constexpr (RESB) {
                    // weights resident: all nine taps x two rows in one commit group, same MMA shape throughout.  The A operand
                    // of tap (r, s) for output row j is patch row rho = r + j; taps are issued by patch row in the order
                    // rho = 1, 2, 0, 3 (both rows read rows 1 and 2), which fixes the accumulation order of every output.
                    acc_fence<2 * kH>(acc);
                    wgmma_fence();
#pragma unroll
                    for (int o = 0; o < 4; o++) {
                        const int rho = o == 0 ? 1 : (o == 1 ? 2 : (o == 2 ? 0 : 3));
#pragma unroll
                        for (int s3 = 0; s3 < 3; s3++) {
                            const uint64_t da = make_desc(a_base + (uint32_t)((rho * kPatchW + s3) * 128));
#pragma unroll
                            for (int j = 0; j < 2; j++) {
                                const int r = rho - j;
                                if (r < 0 || r > 2) continue;
                                const uint64_t db = make_desc(smem_u32(sB + (r * 3 + s3) * Plan::kBBytes));
#pragma unroll
                                for (int k = 0; k < kKC / 16; k++)
                                    wgmma<BN, 0, 0, 0>(acc + j * kH, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (c | o | s3 | k) != 0);
                            }
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    acc_fence<2 * kH>(acc);
                } else {
                    int prevb = -1;
                    for (int tap = 0; tap < 9; tap++) {
                        mbar_wait(&fullB[sb], pb);
                        const int r = tap / 3, s = tap - 3 * r;
                        const uint64_t db = make_desc(smem_u32(sB + sb * Plan::kBBytes));
                        acc_fence<2 * kH>(acc);
                        wgmma_fence();
#pragma unroll
                        for (int j = 0; j < 2; j++) {
                            const uint64_t da = make_desc(a_base + (uint32_t)(((r + j) * kPatchW + s) * 128));
#pragma unroll
                            for (int k = 0; k < kKC / 16; k++)
                                wgmma<BN, 0, 0, 0>(acc + j * kH, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (c | tap | k) != 0);
                        }
                        wgmma_commit();
                        acc_fence<2 * kH>(acc);
                        if (prevb >= 0) {
                            wgmma_wait<1>();
                            release(&emptyB[prevb], lane);
                        }
                        prevb = sb;
                        if (++sb == Plan::kBStages) { sb = 0; pb ^= 1; }
                    }
                    wgmma_wait<0>();
                    acc_fence<2 * kH>(acc);
                    release(&emptyB[prevb], lane);
                }
                release(&emptyA[sa], lane);
                if (++sa == kRowAStages) { sa = 0; pa ^= 1; }
            }
            if (!p.pool) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
#pragma unroll
                    for (int g = 0; g < BN / 64; g++) {
                        if (threadIdx.x == 0) { if (RESB) tma_store_wait_read<0>(); else tma_store_wait_read<1>(); }
                        consumer_sync();
                        uint8_t* ob = out_stage + (RESB ? 0 : obuf * kStageBytes);
                        stage_rows(ob, acc + j * kH + g * 32, p.bias + n0 + g * 64, p.relu, row, lane & 3);
                        fence_proxy_async();
                        consumer_sync();
                        if (threadIdx.x == 0) {
                            tma_store_4d(&map_out, ob, n0 + g * 64, x0, y0 + j, img);
                            tma_store_commit();
                        }
                        obuf ^= 1;
                    }
                }
            } else {
#pragma unroll
                for (int g = 0; g < BN / 64; g++) {
                    if (threadIdx.x == 0) tma_store_wait_read<1>();
                    consumer_sync();
                    uint8_t* ob = out_stage + obuf * (RESB ? kStageBytes / 2 : kStageBytes);  // pooled tile: 64 rows = 8 KB
                    const float* a0 = acc + g * 32;
                    const float* a1 = acc + kH + g * 32;
                    const float* bias = p.bias + n0 + g * 64;
                    const int q = lane & 3;
#pragma unroll
                    for (int i = 0; i < 2; i++) {
                        const int r = row + 8 * i;
                        const int prow = r >> 1;  // pooled pixel within the 64-wide pooled segment
#pragma unroll
                        for (int jj = 0; jj < 8; jj++) {
                            const int c = 8 * jj + 2 * q;
                            // vertical max of the pair (same bias, monotone ReLU / rounding: order is irrelevant)
                            float v0 = fmaxf(a0[4 * jj + 2 * i], a1[4 * jj + 2 * i]) + __ldg(bias + c);
                            float v1 = fmaxf(a0[4 * jj + 2 * i + 1], a1[4 * jj + 2 * i + 1]) + __ldg(bias + c + 1);
                            if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                            uint32_t pk = pack_bf16(v0, v1);
                            uint32_t o1 = __shfl_xor_sync(0xffffffffu, pk, 4);  // horizontal neighbour: pixel r ^ 1
                            __nv_bfloat162 m2 = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&pk), *reinterpret_cast<__nv_bfloat162*>(&o1));
                            if ((lane & 4) == 0)
                                *reinterpret_cast<__nv_bfloat162*>(ob + prow * 128 + ((jj ^ (prow & 7)) << 4) + 4 * q) = m2;
                        }
                    }
                    fence_proxy_async();
                    consumer_sync();
                    if (threadIdx.x == 0) {
                        tma_store_4d(&map_out, ob, n0 + g * 64, x0 >> 1, y0 >> 1, img);
                        tma_store_commit();
                    }
                    obuf ^= 1;
                }
            }
        }
        if (threadIdx.x == 0) tma_store_wait_all();
    }
}

// ---------------------------------------------------------------------------------------------
// First layer (conv1_1, Cin = 3, K = 27 -> 32) on the tensor cores with the im2col done in shared memory:
// warps 8-23 (four groups, round-robin over tiles) build the A tile of an 8x16 pixel tile straight from the uint8 / f32
// image (pre-processing `BGR - PIXEL_MEANS` fused, zero outside the image = SAME padding) in the swizzled K-major
// layout; warps 0-7 are two consumer warpgroups that take the tiles alternately: per tile two halves of 64 pixels,
// each two K = 16 wgmmas against the resident 64 x 64 weight tile, then bf16 pack and TMA store.  No im2col tensor
// ever exists in HBM.
// The layer is a large write with almost no math: per tile the builder (27 dependent-free byte loads) and the
// epilogue are latency chains, so the kernel keeps four builds and two epilogues in flight per SM.
// ---------------------------------------------------------------------------------------------
constexpr int kC1Stages = 6;
constexpr int kC1EpiGroups = 2, kC1BuildGroups = 4;
constexpr int kC1Threads = 128 * (kC1EpiGroups + kC1BuildGroups);  // 8 consumer warps, 16 A-builder warps
constexpr int kC1PatchWords = 10 * 16;   // raw uint8 input patch of a tile: 10 rows x 14 words (+2 pad), per builder group x 2 buffers
constexpr int kC1PatchOff = kC1Stages * kABytes + 64 * 128 + kC1EpiGroups * 2 * kStageBytes;
constexpr int kC1BarOff = kC1PatchOff + kC1BuildGroups * 2 * kC1PatchWords * 4;
constexpr int kC1Smem = kC1BarOff + 256 + 1024;

// Input element types: unsigned char / float = [B,H,W,3] colour image (BGR); DepthIn = [B,H,W] raw depth image (one
// float per pixel, sensor units): the `_p` trunk's input blob clip(d / 2000, 0, 1) * 255 tiled x3 - PIXEL_MEANS
// (lib/fcn/test.py:70-76) is formed on the fly in float32 exactly as numpy forms it.
struct DepthIn { float d; };

// The grey value clip(d / 2000, 0, 1) * 255 of the depth blob, one rounding per numpy operation (the caller subtracts the
// channel mean with __fsub_rn).  k_conv1_tc and k_im2col_c3 both form the blob here, so the conv1_1_p weight gradient sees
// exactly the values the forward MMA consumed.
__device__ __forceinline__ float depth_gray(float d)
{
    return __fmul_rn(fminf(fmaxf(__fdiv_rn(d, 2000.f), 0.f), 1.f), 255.f);
}

template <typename TIn>
__global__ void __launch_bounds__(kC1Threads, 1)
k_conv1_tc(const TIn* __restrict__ in, const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_out,
           const ConvParams p, float m0, float m1, float m2)
{
    constexpr int BN = 64;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sb = smem + kC1Stages * kABytes;          // weights: 64 rows x 128 B, swizzled (TMA)
    uint8_t* out_stage = sb + 64 * 128;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kC1BarOff);
    uint64_t* empty = full + kC1Stages;
    uint64_t* wbar = empty + kC1Stages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
        for (int s = 0; s < kC1Stages; s++) { mbar_init(&full[s], 4); mbar_init(&empty[s], 4); }
        mbar_init(wbar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= 4 * kC1EpiGroups) {
        // ===================== A builders: one tile row (pixel) per thread; the groups take tiles round-robin =====================
        const int group = (threadIdx.x - 128 * kC1EpiGroups) >> 7;
        const int r = (threadIdx.x - 128 * kC1EpiGroups) & 127;
        const int hl = r >> 4, wl = r & 15;
        uint32_t* patch_base = reinterpret_cast<uint32_t*>(smem + kC1PatchOff);
        // aligned-word staging needs word-aligned image rows
        const bool fast_u8 = sizeof(TIn) == 1 && (p.W & 3) == 0 && (reinterpret_cast<uintptr_t>(in) & 3) == 0;
        int it = 0, lit = 0;
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, it++) {
            if (it % kC1BuildGroups != group) continue;
            const int stage = it % kC1Stages;
            const uint32_t phase = (it / kC1Stages) & 1;
            const int tw = tile % p.tiles_w;
            const int rest = tile / p.tiles_w;
            const int th = rest % p.tiles_h, img = rest / p.tiles_h;
            const int y = th * kTileH + hl, x = tw * kTileW + wl;
            constexpr int kInCh = std::is_same<TIn, DepthIn>::value ? 1 : 3;
            const TIn* base = in + (size_t)img * p.H * p.W * kInCh;
            float v[32];
            // K = 27, 28 carry 1.0: the matching weight rows hold the bias (bf16 hi + lo parts, patched into the
            // resident weight tile by the MMA warp), so the bias add happens inside the MMA
            v[27] = 1.f; v[28] = 1.f;
#pragma unroll
            for (int k = 29; k < 32; k++) v[k] = 0.f;
            bool done = false;
            if constexpr (sizeof(TIn) == 1) {
                if (fast_u8) {
                    // uint8 fast path: the tile's raw 10 x 18 px patch is staged once in shared memory with aligned
                    // 32-bit loads -- a patch row starts at byte (16 tw - 1) * 3 = 48 tw - 3 of the image row, so the
                    // 14-word window from byte 48 tw - 4 is word aligned and the patch sits at byte offset 1 in it --
                    // and every thread then cuts its 3 x 9 bytes out of it (3 words + 2 byte-permutes per row) instead
                    // of issuing 27 byte loads with their own address arithmetic and bounds tests.
                    uint32_t* pw = patch_base + (group * 2 + (lit & 1)) * kC1PatchWords;
                    const int y0 = th * kTileH - 1, wq0 = 12 * tw - 1, row_words = (p.W * 3) >> 2;
                    const uint32_t* img32 = reinterpret_cast<const uint32_t*>(base);
                    for (int idx = r; idx < 140; idx += 128) {
                        const int prow = idx / 14, wi = idx - prow * 14;
                        const int yy = y0 + prow, wq = wq0 + wi;
                        uint32_t word = 0;
                        if (yy >= 0 && yy < p.H && wq >= 0 && wq < row_words) word = __ldg(img32 + (size_t)yy * row_words + wq);
                        pw[prow * 16 + wi] = word;
                    }
                    if (group == 0) asm volatile("bar.sync 3, 128;" ::: "memory");
                    else if (group == 1) asm volatile("bar.sync 4, 128;" ::: "memory");
                    else if (group == 2) asm volatile("bar.sync 5, 128;" ::: "memory");
                    else asm volatile("bar.sync 6, 128;" ::: "memory");
                    const int boff = 1 + 3 * wl, w0 = boff >> 2, o = boff & 3;
                    const uint32_t sel = (uint32_t)(o | ((o + 1) << 4) | ((o + 2) << 8) | ((o + 3) << 12));
                    const bool border = th == 0 || th * kTileH + kTileH + 1 > p.H || tw == 0 || tw * kTileW + kTileW + 1 > p.W;
#pragma unroll
                    for (int dy = 0; dy < 3; dy++) {
                        const uint32_t* rowp = pw + (hl + dy) * 16 + w0;
                        const uint32_t a0 = rowp[0], a1 = rowp[1], a2 = rowp[2];
                        const uint32_t b03 = __byte_perm(a0, a1, sel), b47 = __byte_perm(a1, a2, sel), b8 = (a2 >> (8 * o)) & 0xffu;
#pragma unroll
                        for (int k = 0; k < 9; k++) {
                            const uint32_t byte = k < 4 ? (b03 >> (8 * k)) & 0xffu : (k < 8 ? (b47 >> (8 * (k - 4))) & 0xffu : b8);
                            const int c = k % 3;
                            v[dy * 9 + k] = (float)byte - (c == 0 ? m0 : (c == 1 ? m1 : m2));
                        }
                    }
                    if (border) {   // SAME padding pads the mean-subtracted image with zeros
#pragma unroll
                        for (int dy = 0; dy < 3; dy++) {
                            const int yy = y + dy - 1;
#pragma unroll
                            for (int dx = 0; dx < 3; dx++) {
                                const int xx = x + dx - 1;
                                if (!(yy >= 0 && yy < p.H && xx >= 0 && xx < p.W)) {
                                    v[(dy * 3 + dx) * 3 + 0] = 0.f; v[(dy * 3 + dx) * 3 + 1] = 0.f; v[(dy * 3 + dx) * 3 + 2] = 0.f;
                                }
                            }
                        }
                    }
                    lit++;
                    done = true;
                }
            }
            if (!done) {
#pragma unroll
                for (int dy = 0; dy < 3; dy++) {
                    const int yy = y + dy - 1;
                    const bool rowok = yy >= 0 && yy < p.H;
#pragma unroll
                    for (int dx = 0; dx < 3; dx++) {
                        const int xx = x + dx - 1;
                        const bool ok = rowok && xx >= 0 && xx < p.W;
                        if constexpr (std::is_same<TIn, DepthIn>::value) {
                            float g = 0.f;
                            if (ok) g = depth_gray(base[(size_t)yy * p.W + xx].d);
                            v[(dy * 3 + dx) * 3 + 0] = ok ? __fsub_rn(g, m0) : 0.f;
                            v[(dy * 3 + dx) * 3 + 1] = ok ? __fsub_rn(g, m1) : 0.f;
                            v[(dy * 3 + dx) * 3 + 2] = ok ? __fsub_rn(g, m2) : 0.f;
                        } else {
                            const TIn* px = base + ((size_t)yy * p.W + xx) * 3;
                            v[(dy * 3 + dx) * 3 + 0] = ok ? (float)px[0] - m0 : 0.f;
                            v[(dy * 3 + dx) * 3 + 1] = ok ? (float)px[1] - m1 : 0.f;
                            v[(dy * 3 + dx) * 3 + 2] = ok ? (float)px[2] - m2 : 0.f;
                        }
                    }
                }
            }
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem + stage * kABytes + r * 128;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint32_t pk[4];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    __nv_bfloat162 b2 = __floats2bfloat162_rn(v[j * 8 + q * 2], v[j * 8 + q * 2 + 1]);
                    pk[q] = *reinterpret_cast<uint32_t*>(&b2);
                }
                *reinterpret_cast<uint4*>(sa + ((j ^ (r & 7)) << 4)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
            }
            fence_proxy_async();  // generic-proxy writes -> visible to the tensor-core (async proxy) reads
            __syncwarp();
            if (lane == 0) mbar_arrive(&full[stage]);
        }
    } else {
        // ===================== consumer warpgroup eg = warps 4 eg .. 4 eg + 3: the tiles with it & 1 == eg =====================
        const int eg = warp >> 2, wq = warp & 3;
        const bool issuer = (threadIdx.x & 127) == 0;
        // one-time weight load; bias -> weight rows K = 27 (bf16 of the bias) and K = 28 (bf16 of the remainder), swizzled
        // K-major layout: element k of output channel n sits at n * 128 + ((k / 8) ^ (n & 7)) * 16 + (k % 8) * 2
        if (warp == 0) {
            if (elect_one()) {
                mbar_arrive_expect_tx(wbar, 64 * 128);
                tma_load_2d(sb, &map_w, wbar, 0, 0);
            }
            __syncwarp();
            mbar_wait(wbar, 0);   // every lane observes the completed TMA before it patches the tile
            for (int n = lane; n < BN; n += 32) {
                const float bv = p.bias[n];
                const __nv_bfloat16 hi = __float2bfloat16_rn(bv);
                const __nv_bfloat16 lo = __float2bfloat16_rn(bv - __bfloat162float(hi));
                uint8_t* rowp = sb + n * 128 + ((3 ^ (n & 7)) << 4);
                *reinterpret_cast<__nv_bfloat16*>(rowp + 6) = hi;    // k = 27
                *reinterpret_cast<__nv_bfloat16*>(rowp + 8) = lo;    // k = 28
            }
            fence_proxy_async();  // generic-proxy writes -> visible to the wgmma (async proxy) reads
        }
        asm volatile("bar.sync 7, 256;" ::: "memory");
        const uint64_t db = make_desc(smem_u32(sb));
        uint8_t* my_stage = out_stage + eg * 2 * kStageBytes;
        const __nv_bfloat162 floor2 = __floats2bfloat162_rn(p.relu ? 0.f : -INFINITY, p.relu ? 0.f : -INFINITY);
        int it = 0, obuf = 0;
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, it++) {
            if ((it & 1) != eg) continue;
            const int tw = tile % p.tiles_w;
            const int rest = tile / p.tiles_w;
            const int th = rest % p.tiles_h, img = rest / p.tiles_h;
            const int stage = it % kC1Stages;
            mbar_wait(&full[stage], (it / kC1Stages) & 1);
            if (issuer) tma_store_wait_read<1>();         // staging buffer obuf: the store of two tiles ago has read it
            if (eg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
            else asm volatile("bar.sync 2, 128;" ::: "memory");
            uint8_t* ob = my_stage + obuf * kStageBytes;
            const uint32_t sa = smem_u32(smem + stage * kABytes);
#pragma unroll
            for (int half = 0; half < 2; half++) {       // pixels 64 half .. 64 half + 63 of the tile
                float acc[BN / 2];
                acc_fence<BN / 2>(acc);
                wgmma_fence();
                const uint64_t da = make_desc(sa + half * 64 * 128);
                wgmma<BN, 0, 0, 0>(acc, da, db, 0);          // K 0..15
                wgmma<BN, 0, 0, 0>(acc, da + 2, db + 2, 1);  // K 16..31 (27, 28 = bias; 29..31 are zero)
                wgmma_commit();
                wgmma_wait<0>();
                acc_fence<BN / 2>(acc);
                if (half == 1) release(&empty[stage], lane);   // the tile's MMAs are done reading its A stage
                const int q = lane & 3;
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    const int r = half * 64 + wq * 16 + (lane >> 2) + 8 * i;
#pragma unroll
                    for (int jj = 0; jj < 8; jj++) {
                        // bias already inside the accumulator; ReLU on the packed pair (rounding is monotone, 0 is exact)
                        uint32_t pk = pack_bf16(acc[4 * jj + 2 * i], acc[4 * jj + 2 * i + 1]);
                        __nv_bfloat162 b2 = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&pk), floor2);
                        *reinterpret_cast<__nv_bfloat162*>(ob + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * q) = b2;
                    }
                }
            }
            fence_proxy_async();
            if (eg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
            else asm volatile("bar.sync 2, 128;" ::: "memory");
            if (issuer) {
                tma_store_4d(&map_out, ob, 0, tw * kTileW, th * kTileH, img);
                tma_store_commit();
            }
            obuf ^= 1;
        }
        if (issuer) tma_store_wait_all();
    }
}

// ---------------------------------------------------------------------------------------------
// conv1_1 (Cin = 3, K = 27: below any tensor-core tile) on the CUDA cores, fused with the input
// pre-processing-free path: fp32 NHWC in, bf16 NHWC out, bias + ReLU.  One thread = one pixel x 16
// output channels; the 27 x Cout weights sit in shared memory.
// ---------------------------------------------------------------------------------------------
template <int CO_PER_THREAD>
__global__ void __launch_bounds__(256)
k_conv_small_cin(const float* __restrict__ in, const float* __restrict__ w /*[3][3][Cin][Cout]*/,
                 const float* __restrict__ bias, __nv_bfloat16* __restrict__ out, int B, int H, int W, int Cin, int Cout,
                 int relu)
{
    extern __shared__ float sw[];  // [9*Cin][Cout] + bias[Cout]
    const int K = 9 * Cin;
    for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) sw[i] = w[i];
    for (int i = threadIdx.x; i < Cout; i += blockDim.x) sw[K * Cout + i] = bias[i];
    __syncthreads();
    const int groups = Cout / CO_PER_THREAD;
    const size_t total = (size_t)B * H * W * groups;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(idx % groups);
        const size_t pix = idx / groups;
        const int x = (int)(pix % W), y = (int)((pix / W) % H);
        const size_t n = pix / ((size_t)W * H);
        float acc[CO_PER_THREAD];
#pragma unroll
        for (int k = 0; k < CO_PER_THREAD; k++) acc[k] = sw[K * Cout + g * CO_PER_THREAD + k];
        for (int r = 0; r < 3; r++) {
            const int yy = y + r - 1;
            if (yy < 0 || yy >= H) continue;
            for (int s = 0; s < 3; s++) {
                const int xx = x + s - 1;
                if (xx < 0 || xx >= W) continue;
                const float* ip = in + ((n * H + yy) * W + xx) * Cin;
                for (int c = 0; c < Cin; c++) {
                    const float v = __ldg(ip + c);
                    const float* wp = sw + ((r * 3 + s) * Cin + c) * Cout + g * CO_PER_THREAD;
#pragma unroll
                    for (int k = 0; k < CO_PER_THREAD; k++) acc[k] = fmaf(v, wp[k], acc[k]);
                }
            }
        }
        __nv_bfloat16* op = out + pix * Cout + g * CO_PER_THREAD;
#pragma unroll
        for (int k = 0; k < CO_PER_THREAD; k += 2) {
            float v0 = acc[k], v1 = acc[k + 1];
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            *reinterpret_cast<__nv_bfloat162*>(op + k) = __floats2bfloat162_rn(v0, v1);
        }
    }
}

// im2col for the first layer only (Cin = 3, K = 27 < one wgmma K chunk of 64): [B,H,W,3] -> [B,H,W,64] bf16 with
// K index = tap * 3 + c (zero beyond 27), so conv1_1 runs on the tensor cores as a 1x1 convolution.
// The input pre-processing of the caller (lib/fcn/test.py:37-110: BGR - PIXEL_MEANS) is fused for uint8
// input: value = (float)u8 - mean[c].  DepthIn: the depth blob depth_gray(d) - mean[c] of a raw [B,H,W] depth image, the
// values k_conv1_tc<DepthIn> feeds its MMA (the im2col view the conv1_1_p weight gradient reads).
template <typename TIn>
__global__ void __launch_bounds__(256)
k_im2col_c3(const TIn* __restrict__ in, __nv_bfloat16* __restrict__ out, int H, int W, float m0, float m1, float m2)
{
    // grid = (ceil(W / 128), H, B): a CTA builds 128 pixels x 64 K-values of one image row in four 32-pixel passes (614 k tiny
    // CTAs at batch 64 were launch-bound).  The 3 x 130 x 3 input patch (mean subtracted, zero outside the image = SAME padding)
    // is staged in shared memory once; thread (x, j) then packs the 8 K-values k = 8j .. 8j+7 (K order tap*3 + c) into one 16-byte store.
    constexpr int kSeg = 128;
    constexpr int kInCh = std::is_same<TIn, DepthIn>::value ? 1 : 3;
    __shared__ float patch[3][(kSeg + 2) * 3];
    const int y = blockIdx.y, n = blockIdx.z, x0 = blockIdx.x * kSeg, t = threadIdx.x;
    const TIn* img = in + (size_t)n * H * W * kInCh;
    constexpr int kRow = (kSeg + 2) * 3;
    for (int i = t; i < 3 * kRow; i += 256) {
        const int r = i / kRow, rem = i - r * kRow, px = rem / 3, c = rem - px * 3;
        const int yy = y + r - 1, xx = x0 + px - 1;
        float v = 0.f;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            if constexpr (std::is_same<TIn, DepthIn>::value)
                v = __fsub_rn(depth_gray(img[yy * W + xx].d), c == 0 ? m0 : (c == 1 ? m1 : m2));
            else
                v = (float)img[(yy * W + xx) * 3 + c] - (c == 0 ? m0 : (c == 1 ? m1 : m2));
        }
        patch[r][rem] = v;
    }
    __syncthreads();
    const int j = t & 7;
#pragma unroll
    for (int pass = 0; pass < kSeg / 32; pass++) {
        const int xl = pass * 32 + (t >> 3), x = x0 + xl;
        if (x >= W) break;
        __align__(16) __nv_bfloat16 v[8];
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int k = j * 8 + e;  // tap = k / 3 (dy = tap / 3, dx = tap % 3), c = k % 3 -> patch[dy][(xl + dx) * 3 + c]
            float val = 0.f;
            if (k < 27) {
                const int dy = k / 9, rem = k - dy * 9;  // rem = dx * 3 + c
                val = patch[dy][xl * 3 + rem];
            }
            v[e] = __float2bfloat16_rn(val);
        }
        *reinterpret_cast<uint4*>(out + (((size_t)n * H + y) * W + x) * 64 + j * 8) = *reinterpret_cast<const uint4*>(v);
    }
}

// 2x2 / stride 2 max pool, NHWC bf16 (Network.max_pool, network.py:303-310; H, W even here)
__global__ void __launch_bounds__(256)
k_maxpool2x2_bf16(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int B, int H, int W, int C)
{
    const int Ho = H / 2, Wo = W / 2, cg = C / 8;
    const size_t total = (size_t)B * Ho * Wo * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(idx % cg);
        size_t r = idx / cg;
        const int xo = (int)(r % Wo); r /= Wo;
        const int yo = (int)(r % Ho);
        const size_t n = r / Ho;
        const __nv_bfloat16* p0 = in + ((n * H + 2 * yo) * W + 2 * xo) * C + g * 8;
        uint4 a = __ldg(reinterpret_cast<const uint4*>(p0));
        uint4 b = __ldg(reinterpret_cast<const uint4*>(p0 + C));
        uint4 c = __ldg(reinterpret_cast<const uint4*>(p0 + (size_t)W * C));
        uint4 d = __ldg(reinterpret_cast<const uint4*>(p0 + (size_t)W * C + C));
        uint4 o;
        const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a);
        const __nv_bfloat162* pb = reinterpret_cast<const __nv_bfloat162*>(&b);
        const __nv_bfloat162* pc = reinterpret_cast<const __nv_bfloat162*>(&c);
        const __nv_bfloat162* pd = reinterpret_cast<const __nv_bfloat162*>(&d);
        __nv_bfloat162* po = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
        for (int k = 0; k < 4; k++) po[k] = __hmax2(__hmax2(pa[k], pb[k]), __hmax2(pc[k], pd[k]));
        *reinterpret_cast<uint4*>(out + ((n * Ho + yo) * Wo + xo) * C + g * 8) = o;
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int make_map_nhwc(CUtensorMap* m, const void* ptr, int B, int H, int W, int C, int box_c, int box_w = kTileW, int box_h = kTileH)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (driver too old?)"); return PCNN_E_CUDA; }
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(NHWC %dx%dx%dx%d) failed: %d", B, H, W, C, (int)r); return PCNN_E_CUDA; }
    return PCNN_OK;
}

template <int BN, int BM = kTileM>
static int launch_conv(const CUtensorMap& mi, const CUtensorMap& mw, const CUtensorMap& mo, const ConvParams& p, int num_sms,
                       cudaStream_t st)
{
    using Plan = SmemPlan<BN, BM>;
    PCNN_SMEM_OPTIN((k_conv_tc<BN, BM>), Plan::kTotal, "conv_tc");
    int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
    k_conv_tc<BN, BM><<<grid, kThreadsConv, Plan::kTotal, st>>>(mi, mw, mo, p);
    return check_launch("conv_tc");
}

template <int BN, bool RESB>
static int launch_conv_row2(const CUtensorMap& mi, const CUtensorMap& mw, const CUtensorMap& mo, const ConvParams& p, int num_sms,
                            cudaStream_t st)
{
    using Plan = RowPlan<BN, RESB>;
    PCNN_SMEM_OPTIN((k_conv_row2<BN, RESB>), Plan::kTotal, "conv_row2");
    int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
    if (RESB) grid = grid / p.n_tiles_n * p.n_tiles_n;  // every CTA owns one N tile
    k_conv_row2<BN, RESB><<<grid, kThreadsRow, Plan::kTotal, st>>>(mi, mw, mo, p);
    return check_launch("conv_row2");
}

}  // namespace convtc
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::convtc;

// in [B,H,W,Cin] bf16, weights [Cout][ksize*ksize*Cin] bf16 (tap-major, channel-minor), bias [Cout] f32,
// out [B,H,W,Cout] bf16.  Cin % 64 == 0, Cout % 64 == 0, ksize in {1, 3}.
static int conv_bf16_tc_impl(const void* in, const void* weights, const float* bias, void* out, int B, int H, int W, int Cin,
                            int Cout, int ksize, int relu, int block_n, int pool, void* stream);

extern "C" int pcnn_conv_bf16_tc(const void* in, const void* weights, const float* bias, void* out, int B, int H, int W,
                                 int Cin, int Cout, int ksize, int relu, int block_n, void* stream)
{
    return conv_bf16_tc_impl(in, weights, bias, out, B, H, W, Cin, Cout, ksize, relu, block_n, 0, stream);
}

// conv + bias + ReLU + 2x2/2 max pool fused: out is the POOLED tensor [B,H/2,W/2,Cout] bf16 (H, W even)
extern "C" int pcnn_conv_pool_bf16_tc(const void* in, const void* weights, const float* bias, void* out_pooled, int B, int H,
                                      int W, int Cin, int Cout, int ksize, int relu, int block_n, void* stream)
{
    PCNN_REQUIRE(H % 2 == 0 && W % 2 == 0, "conv_pool: needs even H, W (got %d x %d)", H, W);
    return conv_bf16_tc_impl(in, weights, bias, out_pooled, B, H, W, Cin, Cout, ksize, relu, block_n, 1, stream);
}

static int conv_bf16_tc_impl(const void* in, const void* weights, const float* bias, void* out, int B, int H, int W, int Cin,
                            int Cout, int ksize, int relu, int block_n, int pool, void* stream)
{
    PCNN_REQUIRE(in && weights && bias && out, "conv: NULL tensor pointer");
    PCNN_REQUIRE(ksize == 1 || ksize == 3, "conv: ksize must be 1 or 3 (got %d)", ksize);
    PCNN_REQUIRE(Cin % 64 == 0 && Cin >= 64, "conv: Cin must be a multiple of 64 (got %d)", Cin);
    PCNN_REQUIRE(Cout % 64 == 0 && Cout >= 64, "conv: Cout must be a multiple of 64 (got %d)", Cout);
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "conv: bad shape");
    int bn = block_n;
    // default N tile: 256 for the deep layers (K = taps * Cin >= 2304), where it is faster on the H100 (tools/bench_trunk.py prints
    // every such layer at both N tiles); 128 below
    if (bn == 0) bn = Cout % 256 == 0 && ksize * ksize * Cin >= 2304 ? 256 : (Cout % 128 == 0 ? 128 : 64);
    PCNN_REQUIRE((bn == 64 || bn == 128 || bn == 256) && Cout % bn == 0, "conv: block_n %d does not divide Cout %d", bn, Cout);
    int dev = 0, sms = kNumSMs;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap mi, mw, mo;
    int rc;
    // The K-small 3x3 layers (Cin <= 128) take one of two kernels chosen from the shape alone; an explicit block_n always runs
    // the 128-pixel tile kernel at that N tile.
    //   Cout = 128 (conv2_1, conv2_2 (+ pool2), conv2_2's input gradient): the 256-pixel tile (16 x 16) at BN = 128, below.
    //     Batch 32, one H100 SXM at a 400 W power limit (tools/bench_trunk.py): conv2_1 0.758 ms, conv2_2 + pool2 1.334 ms,
    //     against 0.849 / 1.527 ms on the 128-pixel tile at BN = 128 and 0.922 / 1.959 ms in row mode (N = 64).
    //   Cout = 64 (conv1_2, conv2_1's input gradient): row mode (two output rows x 128 px per work item, one A patch per
    //     64-channel chunk reused by all nine taps); conv1_2 keeps its nine 8-KB weight slices resident in shared memory
    //     (conv1_2 + pool1 at batch 32: 1.371 ms, same card and run).
    const bool tile256 = block_n == 0 && ksize == 3 && Cin <= 128 && Cout == 128;
    if (block_n == 0 && ksize == 3 && Cin <= 128 && Cout == 64 && H % 2 == 0 && W >= kRowPx) {
        const bool resb = Cin == 64;
        bn = 64;
        rc = make_map_nhwc(&mi, in, B, H, W, Cin, kKC, kPatchW, kPatchH);
        if (rc) return rc;
        rc = make_map_weights(&mw, weights, 9 * Cin, Cout, bn);
        if (rc) return rc;
        rc = pool ? make_map_nhwc(&mo, out, B, H / 2, W / 2, Cout, 64, kRowPx / 2, 1) : make_map_nhwc(&mo, out, B, H, W, Cout, 64, kRowPx, 1);
        if (rc) return rc;
        ConvParams p;
        p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.ksize = 3; p.taps = 9;
        p.tile_h = 2; p.tile_w = kRowPx;
        p.tiles_h = H / 2;
        p.tiles_w = (W + kRowPx - 1) / kRowPx;
        p.n_tiles_n = Cout / bn;
        p.total_tiles = B * p.tiles_h * p.tiles_w * p.n_tiles_n;
        p.relu = relu; p.pool = pool; p.bias = bias; p.kc_outer = 0;
        if (resb && p.total_tiles >= p.n_tiles_n) return launch_conv_row2<64, true>(mi, mw, mo, p, sms, st);
        return launch_conv_row2<64, false>(mi, mw, mo, p, sms, st);
    }
    // pixel tile: 8 x 16, or 16 x 8 when that covers the map with fewer tiles (conv5: 30 x 40 -> 10 tiles instead of 12);
    // 16 x 16 for the 256-pixel tile.  The tile's pixel order is whatever the TMA box says (row = h * tile_w + w for load
    // and store alike), so only the box shape and the tile origin change; the epilogue stores (and pools) one 128-pixel
    // half at a time, and the fused pool is written for 8 x 16 halves.
    int tile_h = kTileH, tile_w = kTileW;
    if (tile256) tile_h = 2 * kTileH;
    else if (!pool && ((H + 15) / 16) * ((W + 7) / 8) < ((H + 7) / 8) * ((W + 15) / 16)) { tile_h = 16; tile_w = 8; }
    rc = make_map_nhwc(&mi, in, B, H, W, Cin, kKC, tile_w, tile_h);
    if (rc) return rc;
    rc = make_map_weights(&mw, weights, ksize * ksize * Cin, Cout, bn);
    if (rc) return rc;
    rc = pool ? make_map_nhwc(&mo, out, B, H / 2, W / 2, Cout, 64, kTileW / 2, kTileH / 2)
              : make_map_nhwc(&mo, out, B, H, W, Cout, 64, tile_w, tile256 ? kTileH : tile_h);
    if (rc) return rc;
    ConvParams p;
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
    p.ksize = ksize; p.taps = ksize * ksize;
    p.tile_h = tile_h; p.tile_w = tile_w;
    p.tiles_h = (H + tile_h - 1) / tile_h;
    p.tiles_w = (W + tile_w - 1) / tile_w;
    p.n_tiles_n = Cout / bn;
    p.total_tiles = B * p.tiles_h * p.tiles_w * p.n_tiles_n;
    p.relu = relu;
    p.pool = pool;
    p.bias = bias;
    // 256-pixel tile: chunk-outer where these shapes ran in row mode before (even H, W >= 128: every conv2_x shape of a
    // 480 x 640 input), tap-outer where they ran on the 128-pixel tile, so that every call sums in the order it did then and
    // gives the same bits (for Cin = 64 the two orders coincide)
    p.kc_outer = tile256 && H % 2 == 0 && W >= kRowPx;
    if (tile256) return launch_conv<128, 256>(mi, mw, mo, p, sms, st);
    if (bn == 256) return launch_conv<256>(mi, mw, mo, p, sms, st);
    if (bn == 128) return launch_conv<128>(mi, mw, mo, p, sms, st);
    return launch_conv<64>(mi, mw, mo, p, sms, st);
}

// conv with tiny Cin (conv1_1): in [B,H,W,Cin] f32, weights HWIO [3,3,Cin,Cout] f32, out [B,H,W,Cout] bf16
extern "C" int pcnn_conv3x3_small_cin(const float* in, const float* weights_hwio, const float* bias, void* out, int B, int H,
                                      int W, int Cin, int Cout, int relu, void* stream)
{
    PCNN_REQUIRE(in && weights_hwio && bias && out, "conv_small: NULL tensor pointer");
    PCNN_REQUIRE(Cin >= 1 && Cin <= 8 && Cout % 16 == 0 && Cout <= 128, "conv_small: needs Cin <= 8, Cout %% 16 == 0, Cout <= 128");
    size_t smem = sizeof(float) * (size_t)(9 * Cin + 1) * Cout;
    size_t total = (size_t)B * H * W * (Cout / 16);
    int blocks = (int)((total + 255) / 256 < (size_t)kNumSMs * 8 ? (total + 255) / 256 : (size_t)kNumSMs * 8);
    k_conv_small_cin<16><<<blocks, 256, smem, (cudaStream_t)stream>>>(in, weights_hwio, bias, (__nv_bfloat16*)out, B, H, W, Cin,
                                                                      Cout, relu);
    return check_launch("conv_small_cin");
}

extern "C" int pcnn_maxpool2x2_bf16(const void* in, void* out, int B, int H, int W, int C, void* stream)
{
    PCNN_REQUIRE(in && out, "maxpool: NULL tensor pointer");
    PCNN_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "maxpool: needs even H, W and C %% 8 == 0 (got %d,%d,%d)", H, W, C);
    size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 8);
    int blocks = (int)((total + 255) / 256 < (size_t)kNumSMs * 16 ? (total + 255) / 256 : (size_t)kNumSMs * 16);
    k_maxpool2x2_bf16<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, (__nv_bfloat16*)out, B, H, W, C);
    return check_launch("maxpool2x2");
}

// first-layer im2col: in [B,H,W,3] (f32, or u8 with the per-channel mean subtracted) -> out [B,H,W,64] bf16
extern "C" int pcnn_im2col_c3(const void* in, int in_is_u8, const float* mean3_host, void* out_bf16, int B, int H, int W,
                              void* stream)
{
    PCNN_REQUIRE(in && out_bf16, "im2col: NULL tensor pointer");
    float m0 = 0.f, m1 = 0.f, m2 = 0.f;
    if (mean3_host) { m0 = mean3_host[0]; m1 = mean3_host[1]; m2 = mean3_host[2]; }
    PCNN_REQUIRE(H <= 65535 && B <= 65535, "im2col: image too tall for the launch grid");
    dim3 grid((W + 127) / 128, H, B);
    cudaStream_t st = (cudaStream_t)stream;
    if (in_is_u8)
        k_im2col_c3<unsigned char><<<grid, 256, 0, st>>>((const unsigned char*)in, (__nv_bfloat16*)out_bf16, H, W, m0, m1, m2);
    else
        k_im2col_c3<float><<<grid, 256, 0, st>>>((const float*)in, (__nv_bfloat16*)out_bf16, H, W, m0, m1, m2);
    return check_launch("im2col_c3");
}

// first-layer im2col of the depth trunk: a raw depth image [B,H,W] f32 (sensor units) -> [B,H,W,64] bf16 of its blob
// clip(d / 2000, 0, 1) * 255 tiled x3 - mean (lib/fcn/test.py:70-76), the view the conv1_1_p weight gradient reads
extern "C" int pcnn_im2col_depth(const float* depth, const float* mean3_host, void* out_bf16, int B, int H, int W, void* stream)
{
    PCNN_REQUIRE(depth && out_bf16, "im2col_depth: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "im2col_depth: bad shape (%d,%d,%d)", B, H, W);
    PCNN_REQUIRE(H <= 65535 && B <= 65535, "im2col_depth: image too tall for the launch grid");
    float m0 = 0.f, m1 = 0.f, m2 = 0.f;
    if (mean3_host) { m0 = mean3_host[0]; m1 = mean3_host[1]; m2 = mean3_host[2]; }
    dim3 grid((W + 127) / 128, H, B);
    k_im2col_c3<DepthIn><<<grid, 256, 0, (cudaStream_t)stream>>>((const DepthIn*)depth, (__nv_bfloat16*)out_bf16, H, W, m0, m1, m2);
    return check_launch("im2col_depth");
}

// conv1_1 fused: in [B,H,W,3] (u8 minus mean, or f32), weights [64][64] bf16 in im2col K order (tap*3 + c, zero padded),
// bias [64] f32 -> out [B,H,W,64] bf16.  Replaces pcnn_im2col_c3 + a 1x1 pcnn_conv_bf16_tc without the HBM round trip.
static int conv1_fused_impl(const void* in, int in_kind, const float* mean3_host, const void* weights_bf16,
                            const float* bias, void* out_bf16, int B, int H, int W, int relu, void* stream);

extern "C" int pcnn_conv1_fused_tc(const void* in, int in_is_u8, const float* mean3_host, const void* weights_bf16,
                                   const float* bias, void* out_bf16, int B, int H, int W, int relu, void* stream)
{
    return conv1_fused_impl(in, in_is_u8 ? 1 : 0, mean3_host, weights_bf16, bias, out_bf16, B, H, W, relu, stream);
}

// conv1_1_p on a raw depth image [B,H,W] f32 (sensor units): the depth blob of lib/fcn/test.py:70-76 fused into the loader
extern "C" int pcnn_conv1_depth_fused_tc(const float* depth, const float* mean3_host, const void* weights_bf16,
                                         const float* bias, void* out_bf16, int B, int H, int W, int relu, void* stream)
{
    return conv1_fused_impl(depth, 2, mean3_host, weights_bf16, bias, out_bf16, B, H, W, relu, stream);
}

static int conv1_fused_impl(const void* in, int in_kind, const float* mean3_host, const void* weights_bf16,
                                   const float* bias, void* out_bf16, int B, int H, int W, int relu, void* stream)
{
    PCNN_REQUIRE(in && weights_bf16 && bias && out_bf16, "conv1: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "conv1: bad shape");
    float m0 = 0.f, m1 = 0.f, m2 = 0.f;
    if (mean3_host) { m0 = mean3_host[0]; m1 = mean3_host[1]; m2 = mean3_host[2]; }
    CUtensorMap mw, mo;
    int rc = make_map_weights(&mw, weights_bf16, 64, 64, 64);
    if (rc) return rc;
    rc = make_map_nhwc(&mo, out_bf16, B, H, W, 64, 64);
    if (rc) return rc;
    ConvParams p;
    p.B = B; p.H = H; p.W = W; p.Cin = 3; p.Cout = 64; p.ksize = 3; p.taps = 9;
    p.tile_h = kTileH; p.tile_w = kTileW;
    p.tiles_h = (H + kTileH - 1) / kTileH;
    p.tiles_w = (W + kTileW - 1) / kTileW;
    p.n_tiles_n = 1;
    p.total_tiles = B * p.tiles_h * p.tiles_w;
    p.relu = relu; p.pool = 0; p.bias = bias; p.kc_outer = 0;
    int dev = 0, sms = kNumSMs;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int grid = p.total_tiles < sms ? p.total_tiles : sms;
    cudaStream_t st = (cudaStream_t)stream;
    PCNN_SMEM_OPTIN(k_conv1_tc<unsigned char>, kC1Smem, "conv1_tc<u8>");
    PCNN_SMEM_OPTIN(k_conv1_tc<float>, kC1Smem, "conv1_tc<f32>");
    PCNN_SMEM_OPTIN(k_conv1_tc<DepthIn>, kC1Smem, "conv1_tc<depth>");
    if (in_kind == 1) k_conv1_tc<unsigned char><<<grid, kC1Threads, kC1Smem, st>>>((const unsigned char*)in, mw, mo, p, m0, m1, m2);
    else if (in_kind == 2) k_conv1_tc<DepthIn><<<grid, kC1Threads, kC1Smem, st>>>((const DepthIn*)in, mw, mo, p, m0, m1, m2);
    else k_conv1_tc<float><<<grid, kC1Threads, kC1Smem, st>>>((const float*)in, mw, mo, p, m0, m1, m2);
    return check_launch("conv1_fused_tc");
}
