// wgrad_tc.cu — weight gradients of the convolution / fully connected layers on the sm_90a tensor cores, and the
// element-wise halves of the backward pass (ReLU mask, max-pool routing, bias gradients).
//
// Behavioural spec: the gradients TensorFlow derives for Network.conv / Network.fc / Network.max_pool
// (lib/networks/network.py:159-188, 303-310, 392-422) in the training graph of lib/fcn/train.py:206-260:
//   y = relu(conv(x, W) + b)      dz = dy * [y > 0]      dW[r,s,ci,co] = sum_{n,h,w} x[n, h+r-1, w+s-1, ci] * dz[n,h,w,co]
//   db[co] = sum dz[..., co]       dx = conv(dz, W flipped / transposed)   (the forward kernel, conv.hwio_to_tc_dgrad)
//
// Weight gradient as a GEMM whose REDUCTION dimension is the pixel index:
//      dW_tap[co, ci] = sum_p  dZ[p, co] * X[p + tap offset, ci]
// Both operands are NHWC activation tiles exactly as TMA delivers them — 64 pixels x 64 channels, rows of 128 B,
// SWIZZLE_128B — i.e. "MN-major" wgmma operands (the M / N index is the contiguous one, the K index = pixel is the row):
// no transposed copy of any activation is ever made.  One box {64 ch, bw, bh, 1} of dZ at the tile origin and one box
// of X at the origin shifted by the tap (out-of-image = zero = SAME padding) have the same pixel order, so row p of one
// pairs with row p of the other.  Two consumer warpgroups take one 64-channel dZ block each (wgmma M = 64), N <= 256
// (B blocks LBO apart), K = 16 pixels per instruction, FP32 accumulation in registers.
//
//   work item  = (pixel range s, tap group, Cin tile, Cout tile) — for Cin <= 128 up to four taps share one MMA as extra N blocks
//                (N = 256 instead of 64); items of one pixel range are adjacent in launch order so
//                that the 9 taps x tiles that re-read the same activations run together and hit in L2
//   split-K    = the pixel ranges; partial [split][tap][Cout][Cin] fp32 in a workspace, fixed-order reduction
//                (k_wgrad_finish) -> dW in the tensor-core weight layout [Cout][tap * Cin + ci] fp32
#include <float.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace pcnn {
namespace wgtc {

using namespace pcnn::convtc;

constexpr int kWgPx = 64;                          // pixels per K tile
constexpr int kWgBlk = kWgPx * 128;                // one 64-channel block of a tile: 8 KB
constexpr int kWgMaxNB = 4;                        // N <= 256
constexpr int kWgStage = (2 + kWgMaxNB) * kWgBlk;  // 48 KB
constexpr int kWgStages = 4;
constexpr int kWgBarOff = kWgStages * kWgStage;
constexpr int kWgSmem = kWgBarOff + 256 + 1024;
constexpr int kWgThreads = 288;                  // warps 0-7: two consumer warpgroups (dZ channel blocks), warp 8 TMA producer

struct WgParams {
    int B, H, W, Cin, Cout, ksize, taps;
    int bw, bh;                 // pixel box (bw * bh = 64)
    int tiles_w, tiles_h, ktiles;          // K tiles = B * tiles_h * tiles_w
    int ktiles_per_split, splits;
    int n_tile, n_tiles, m_tiles;          // N tile (64 / 128 / 256), Cin / n_tile, ceil(Cout / 128)
    int f16;                               // operands are FP16 (the fully connected head) instead of BF16
    int tg, tap_groups;                    // taps per work item (Cin <= 128: several taps share one MMA as extra N blocks), ceil(taps / tg)
    // splits == 1 (the fully connected layers: more (Cout, Cin) tiles than two waves of CTAs): the epilogue writes the finished
    // gradient dW[co][tap * Cin + ci] = scale * acc (+ decay * w) itself; no partial buffer, no k_wgrad_finish pass
    int direct;
    // Cout = Cin = 64, 3x3 (conv1_2): a 64-channel dZ block fills only half of the M = 128 operand.  The upper half then holds the SAME
    // dZ channels one image row further down (box origin h0 + 1): D[64 + co, tap (2, s)] = sum_p dZ[p + (1, 0), co] X[p + (1, s - 1)] =
    // dW[tap (1, s)] — the item with the B blocks of taps (2, 0..2) (N = 192) produces taps (2, s) in lanes 0..63 and taps (1, s) in
    // lanes 64..127; a second item does taps (0, s) with a zero upper half.  Two N = 192 items instead of three (N = 256, 256, 64):
    // 192 instead of 340 MMA clocks per 16 pixels.  The tile grid starts at image row -1 so that row 0 of dZ meets the upper half.
    int pair64, h_org;
    float scale, decay;
    const float* w;
    float* dW;
};

// Consumer warpgroup wg: D[64 channels of dZ block wg, N] over the item's pixel tiles, then the epilogue from registers.
// Both operands are MN-major (wgmma transpose flags): K rows of 128 B (64 channels), 8-row groups 1024 B apart (SBO),
// 64-channel blocks kWgBlk bytes apart (LBO).
template <int N, int F16>
__device__ __forceinline__ void wgrad_consume(uint8_t* smem, uint64_t* full, uint64_t* empty, int nk, const WgParams& p,
                                              float* __restrict__ partial, int split, int m0, int n0, int tap0, int cb, bool upper,
                                              int wg, int wq, int lane)
{
    float acc[N / 2];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int k = 0; k < nk; k++) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * kWgStage) + wg * kWgBlk;
        const uint32_t sb = smem_u32(smem + stage * kWgStage) + 2 * kWgBlk;
        acc_fence<N / 2>(acc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kWgPx / 16; kk++) {      // 16 pixel rows = 2048 B per K step
            const uint64_t da = make_desc_lbo(sa + kk * 2048, kWgBlk), db = make_desc_lbo(sb + kk * 2048, kWgBlk);
            wgmma<N, F16, 1, 1>(acc, da, db, (k | kk) != 0);
        }
        wgmma_commit();
        acc_fence<N / 2>(acc);
        if (prev >= 0) {
            wgmma_wait<1>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == kWgStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence<N / 2>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
    // accumulator row = output channel of the tile, column = B column (block j / 8 = tap and input-channel block)
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int co = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i - (upper ? 64 : 0);   // upper: the same channels, tap - 3
        if (co >= p.Cout) continue;
#pragma unroll
        for (int j = 0; j < N / 8; j++) {
            const int jb = j / 8;
            const int tap = tap0 + jb / cb - (upper ? 3 : 0), ci = n0 + 64 * (jb % cb) + 8 * (j % 8) + 2 * (lane & 3);
            float2 v = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
            if (p.direct) {
                const size_t o = ((size_t)co * p.taps + tap) * p.Cin + ci;
                v.x *= p.scale; v.y *= p.scale;
                if (p.w) {
                    const float2 wv = __ldg(reinterpret_cast<const float2*>(p.w + o));
                    v.x = fmaf(p.decay, wv.x, v.x); v.y = fmaf(p.decay, wv.y, v.y);
                }
                *reinterpret_cast<float2*>(p.dW + o) = v;
            } else {
                *reinterpret_cast<float2*>(partial + (((size_t)split * p.taps + tap) * p.Cout + co) * p.Cin + ci) = v;
            }
        }
    }
}

// NB = B blocks per stage (wgmma N = 64 NB), the same for every item of a launch: the launch covers the tap groups
// tg_lo .. tg_lo + tg_count - 1 (wgrad_impl launches the full groups and a shorter last group separately)
template <int NB, int F16>
__global__ void __launch_bounds__(kWgThreads, 1)
k_wgrad_tc(const __grid_constant__ CUtensorMap map_x /*[B,H,W,Cin] box {64,bw,bh,1}*/,
           const __grid_constant__ CUtensorMap map_dz /*[B,H,W,Cout] box {64,bw,bh,1}*/, float* __restrict__ partial, const WgParams p,
           int tg_lo, int tg_count)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kWgBarOff);
    uint64_t* empty = full + kWgStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // item -> (split, tap group, n tile, m tile); m fastest
    int item = blockIdx.x;
    const int mt = item % p.m_tiles; item /= p.m_tiles;
    const int nt = item % p.n_tiles; item /= p.n_tiles;
    const int tgi = tg_lo + item % tg_count;
    const int split = item / tg_count;
    const int k_lo = split * p.ktiles_per_split, k_hi = min(k_lo + p.ktiles_per_split, p.ktiles);
    const int nk = k_hi - k_lo;
    const int m0 = mt * 128, n0 = nt * p.n_tile;
    const int tap0 = p.pair64 ? (tgi == 0 ? 6 : 0) : tgi * p.tg;
    const bool up_shift = p.pair64 && tgi == 0;         // upper A block = dZ one row down (see WgParams::pair64)
    const int cb = p.n_tile / 64;                       // 64-channel B blocks per tap
    constexpr int nb = NB;                              // block j = (tap0 + j / cb, channels n0 + 64 (j % cb))
    const bool a2 = m0 + 64 < p.Cout;                   // second 64-channel block of dZ exists
    const bool wg1 = a2 || up_shift;                    // the second consumer warpgroup has a dZ block (else it exits at once)
    const int pad = p.ksize / 2;

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_dz) : "memory");
        for (int s = 0; s < kWgStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], wg1 ? 8 : 4); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t tx = (uint32_t)((wg1 ? 2 : 1) + nb) * kWgBlk;
            int bdx[kWgMaxNB], bdy[kWgMaxNB], bch[kWgMaxNB];       // per B block: tap offset and channel origin (loop invariant)
#pragma unroll
            for (int j = 0; j < kWgMaxNB; j++) {
                const int tap = tap0 + j / cb;
                bdy[j] = tap / p.ksize - pad; bdx[j] = tap % p.ksize - pad; bch[j] = n0 + 64 * (j % cb);
            }
            for (int k = 0; k < nk; k++) {
                int kt = k_lo + k;
                const int tw = kt % p.tiles_w; kt /= p.tiles_w;
                const int th = kt % p.tiles_h;
                const int img = kt / p.tiles_h;
                const int w0 = tw * p.bw, h0 = th * p.bh + p.h_org;
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* st = smem + stage * kWgStage;
                mbar_arrive_expect_tx(&full[stage], tx);
                tma_load_4d(st, &map_dz, &full[stage], m0, w0, h0, img);
                if (a2) tma_load_4d(st + kWgBlk, &map_dz, &full[stage], m0 + 64, w0, h0, img);
                else if (up_shift) tma_load_4d(st + kWgBlk, &map_dz, &full[stage], m0, w0, h0 + 1, img);
#pragma unroll
                for (int j = 0; j < kWgMaxNB; j++)
                    if (j < nb) tma_load_4d(st + (2 + j) * kWgBlk, &map_x, &full[stage], bch[j], w0 + bdx[j], h0 + bdy[j], img);
                if (++stage == kWgStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        const int wg = warp >> 2, wq = warp & 3;
        if (wg == 1 && !wg1) return;
        wgrad_consume<64 * NB, F16>(smem, full, empty, nk, p, partial, split, m0, n0, tap0, cb, up_shift && wg == 1, wg, wq, lane);
    }
}

// dW[co][tap * Cin + ci] = scale * sum_s partial[s][tap][co][ci] (+ decay * w[co][tap * Cin + ci]: l2_regularizer, network.py:171-172)
__global__ void __launch_bounds__(256)
k_wgrad_finish(const float* __restrict__ partial, int splits, int taps, int Cout, int Cin, float scale, const float* __restrict__ w,
               float decay, float* __restrict__ dW)
{
    const size_t per = (size_t)taps * Cout * Cin;
    const size_t n4 = per / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e = 4 * i;                         // element (tap, co, ci..ci+3) of a partial
        const int ci = (int)(e % Cin);
        const size_t r = e / Cin;
        const int co = (int)(r % Cout), tap = (int)(r / Cout);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < splits; s++) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(partial + (size_t)s * per) + i);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        const size_t o = (size_t)co * taps * Cin + (size_t)tap * Cin + ci;
        float4 out = make_float4(acc.x * scale, acc.y * scale, acc.z * scale, acc.w * scale);
        if (w) {
            const float4 wv = __ldg(reinterpret_cast<const float4*>(w + o));
            out.x = fmaf(decay, wv.x, out.x); out.y = fmaf(decay, wv.y, out.y); out.z = fmaf(decay, wv.z, out.z); out.w = fmaf(decay, wv.w, out.w);
        }
        *reinterpret_cast<float4*>(dW + o) = out;
    }
}

// ---------------------------------------------------------------------------------------------
// element-wise backward pieces (bf16 NHWC activations, channels % 8 == 0)
//   k_relu_bwd           dz = g * [y > 0]                                  (+ per-CTA bias-gradient partials)
//   k_maxpool_relu_bwd   dz[n, 2h+i, 2w+j, c] = g[n,h,w,c] at the window's first maximum (raster order) if that y > 0
// Bias gradient: every CTA owns a fixed set of pixels, accumulates its per-channel sums in fp32 and writes them to
// bias_partial[cta][C]; k_bias_finish adds the CTAs in index order.  Every sum has a fixed order (run-to-run deterministic).
// ---------------------------------------------------------------------------------------------
constexpr int kEwThreads = 256;

// The grid-stride step (grid * kEwThreads, ew_grid) is a multiple of the channel-group count C / 8, so a thread always meets the
// SAME 8 channels, group (blockIdx.x * kEwThreads + threadIdx.x) % cg: it sums them in registers.  The CTA partial of a channel
// is then the sum of its threads' registers in thread order (no shared-memory atomics, whose order varies from run to run).
__device__ __forceinline__ void bias_cta_partial(const float racc[8], int C, float* __restrict__ out /*[C]*/)
{
    __shared__ float s_part[kEwThreads * 8];
#pragma unroll
    for (int j = 0; j < 8; j++) s_part[threadIdx.x * 8 + j] = racc[j];
    __syncthreads();
    const int cg = C / 8;
    const int first = (int)(((size_t)blockIdx.x * kEwThreads) % cg);    // channel group of thread 0
    for (int c = threadIdx.x; c < C; c += kEwThreads) {
        int t = (c >> 3) - first;
        if (t < 0) t += cg;
        float s = 0.f;
        for (; t < kEwThreads; t += cg) s += s_part[t * 8 + (c & 7)];
        out[c] = s;
    }
}

__global__ void __launch_bounds__(kEwThreads)
k_relu_bwd(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ y, size_t npix, int C, int has_relu,
           __nv_bfloat16* __restrict__ dz, float* __restrict__ bias_partial /*[grid][C] or null*/)
{
    const int cg = C / 8;
    const size_t total = npix * cg;
    const size_t step = (size_t)gridDim.x * blockDim.x;
    float racc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) racc[j] = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
        const uint4 gv = __ldg(reinterpret_cast<const uint4*>(g) + i);
        uint4 ov = gv;
        if (has_relu) {
            const uint4 yv = __ldg(reinterpret_cast<const uint4*>(y) + i);
            const __nv_bfloat16* yp = reinterpret_cast<const __nv_bfloat16*>(&yv);
            __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(&ov);
#pragma unroll
            for (int j = 0; j < 8; j++)
                if (!(__bfloat162float(yp[j]) > 0.f)) op[j] = __float2bfloat16_rn(0.f);
        }
        if (dz) reinterpret_cast<uint4*>(dz)[i] = ov;
        if (bias_partial) {
            const __nv_bfloat16* op = reinterpret_cast<const __nv_bfloat16*>(&ov);
#pragma unroll
            for (int j = 0; j < 8; j++) racc[j] += __bfloat162float(op[j]);
        }
    }
    if (bias_partial) bias_cta_partial(racc, C, bias_partial + (size_t)blockIdx.x * C);
}

__global__ void __launch_bounds__(kEwThreads)
k_maxpool_relu_bwd(const __nv_bfloat16* __restrict__ g /*[B,H/2,W/2,C]*/, const __nv_bfloat16* __restrict__ y /*[B,H,W,C]*/, int B, int H,
                   int W, int C, __nv_bfloat16* __restrict__ dz /*[B,H,W,C]*/, float* __restrict__ bias_partial)
{
    const int Ho = H / 2, Wo = W / 2, cg = C / 8;
    const size_t total = (size_t)B * Ho * Wo * cg;
    float racc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) racc[j] = 0.f;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int gch = (int)(idx % cg);
        size_t r = idx / cg;
        const int xo = (int)(r % Wo); r /= Wo;
        const int yo = (int)(r % Ho);
        const size_t n = r / Ho;
        const size_t base = ((n * H + 2 * yo) * W + 2 * xo) * C + gch * 8;
        const size_t offs[4] = {base, base + C, base + (size_t)W * C, base + (size_t)W * C + C};
        uint4 yv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) yv[k] = __ldg(reinterpret_cast<const uint4*>(y + offs[k]));
        const uint4 gv = __ldg(reinterpret_cast<const uint4*>(g + ((n * Ho + yo) * Wo + xo) * C + gch * 8));
        const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(&gv);
        uint4 ov[4];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            float best = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(&yv[0])[j]);
            int bi = 0;
#pragma unroll
            for (int k = 1; k < 4; k++) {
                const float v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(&yv[k])[j]);
                if (v > best) { best = v; bi = k; }
            }
            const bool pass = best > 0.f;             // ReLU mask of the conv below the pool (y is post-ReLU)
#pragma unroll
            for (int k = 0; k < 4; k++)
                reinterpret_cast<__nv_bfloat16*>(&ov[k])[j] = (pass && k == bi) ? gp[j] : __float2bfloat16_rn(0.f);
            if (pass) racc[j] += __bfloat162float(gp[j]);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) *reinterpret_cast<uint4*>(dz + offs[k]) = ov[k];
    }
    if (bias_partial) bias_cta_partial(racc, C, bias_partial + (size_t)blockIdx.x * C);
}

// db[c] = scale * sum_k partial[k][c] (+ decay * b[c]); block = 32 channels x 8 row groups, groups combined in fixed order
__global__ void __launch_bounds__(256)
k_bias_finish(const float* __restrict__ partial, int nblocks, int C, float scale, const float* __restrict__ b, float decay,
              float* __restrict__ db)
{
    __shared__ float s[8][33];
    const int cl = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + cl;
    float acc = 0.f;
    if (c < C)
        for (int k = grp; k < nblocks; k += 8) acc += partial[(size_t)k * C + c];
    s[grp][cl] = acc;
    __syncthreads();
    if (grp == 0 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int q = 0; q < 8; q++) t += s[q][cl];
        t *= scale;
        if (b) t = fmaf(decay, b[c], t);     // weight decay is applied to the biases as well (network.py:184)
        db[c] = t;
    }
}

// out (bf16) = a (bf16) + b (bf16 or f32): gradient fan-in of conv4_3 / conv5_3 (score head + vertex head + RoiPoolGrad + trunk)
__global__ void __launch_bounds__(256)
k_add_to_bf16(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, const float* __restrict__ bf, size_t n8,
              __nv_bfloat16* __restrict__ out)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
        float v[8];
        const uint4 av = __ldg(reinterpret_cast<const uint4*>(a) + i);
        const __nv_bfloat16* ap = reinterpret_cast<const __nv_bfloat16*>(&av);
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = __bfloat162float(ap[j]);
        if (b) {
            const uint4 bv = __ldg(reinterpret_cast<const uint4*>(b) + i);
            const __nv_bfloat16* bp = reinterpret_cast<const __nv_bfloat16*>(&bv);
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] += __bfloat162float(bp[j]);
        }
        if (bf) {
            const float4 f0 = __ldg(reinterpret_cast<const float4*>(bf) + 2 * i), f1 = __ldg(reinterpret_cast<const float4*>(bf) + 2 * i + 1);
            v[0] += f0.x; v[1] += f0.y; v[2] += f0.z; v[3] += f0.w; v[4] += f1.x; v[5] += f1.y; v[6] += f1.z; v[7] += f1.w;
        }
        uint4 ov;
        __nv_bfloat162* op = reinterpret_cast<__nv_bfloat162*>(&ov);
#pragma unroll
        for (int j = 0; j < 4; j++) op[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
        reinterpret_cast<uint4*>(out)[i] = ov;
    }
}

static int make_map_nhwc_box(CUtensorMap* m, const void* ptr, int B, int H, int W, int C, int box_w, int box_h)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (driver too old?)"); return PCNN_E_CUDA; }
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(wgrad %dx%dx%dx%d) failed: %d", B, H, W, C, (int)r); return PCNN_E_CUDA; }
    return PCNN_OK;
}

static int plan(int B, int H, int W, int Cin, int Cout, int ksize, WgParams* p)
{
    p->f16 = 0;
    p->B = B; p->H = H; p->W = W; p->Cin = Cin; p->Cout = Cout; p->ksize = ksize; p->taps = ksize * ksize;
    // pixel box: 16 x 4 for images, 64 x 1 for "row lists" (H == 1: fully connected layers), 8 x 8 for narrow maps
    if (H == 1) { p->bw = 64; p->bh = 1; }
    else if (W >= 16) { p->bw = 16; p->bh = 4; }
    else { p->bw = 8; p->bh = 8; }
    p->tiles_w = (W + p->bw - 1) / p->bw;
    p->tiles_h = (H + p->bh - 1) / p->bh;
    p->ktiles = B * p->tiles_h * p->tiles_w;
    p->n_tile = Cin % 256 == 0 ? 256 : (Cin % 128 == 0 ? 128 : 64);
    p->n_tiles = Cin / p->n_tile;
    p->m_tiles = (Cout + 127) / 128;
    // Cin <= 128: N = Cin alone would issue small (N = 64 / 128) MMAs; several taps ride in one instruction as extra N blocks
    p->tg = (p->n_tiles == 1 && p->n_tile < 256 && p->taps > 1) ? 256 / p->n_tile : 1;
    p->tap_groups = (p->taps + p->tg - 1) / p->tg;
    p->pair64 = 0; p->h_org = 0;
    if (Cout == 64 && Cin == 64 && ksize == 3 && H > 1) {
        p->pair64 = 1; p->h_org = -1; p->tg = 3; p->tap_groups = 2;
        p->tiles_h = (H + 1 + p->bh - 1) / p->bh;
        p->ktiles = B * p->tiles_h * p->tiles_w;
    }
    const int base = p->tap_groups * p->n_tiles * p->m_tiles;
    int want = (2 * kNumSMs) / base;                     // just under two full waves of work items (no third, nearly empty wave)
    if (want < 1) want = 1;
    if (want > p->ktiles) want = p->ktiles;
    p->ktiles_per_split = (p->ktiles + want - 1) / want;
    p->splits = (p->ktiles + p->ktiles_per_split - 1) / p->ktiles_per_split;
    p->direct = 0; p->scale = 1.f; p->decay = 0.f; p->w = nullptr; p->dW = nullptr;
    return PCNN_OK;
}

}  // namespace wgtc
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::wgtc;

extern "C" int pcnn_conv_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, size_t* bytes)
{
    PCNN_REQUIRE(bytes && B >= 1 && H >= 1 && W >= 1 && Cin >= 64 && Cin % 64 == 0 && Cout >= 64 && Cout % 64 == 0 && (ksize == 1 || ksize == 3),
                 "conv_wgrad: need Cin, Cout multiples of 64 and ksize 1 or 3 (got %d, %d, %d)", Cin, Cout, ksize);
    WgParams p;
    plan(B, H, W, Cin, Cout, ksize, &p);
    *bytes = align_up(sizeof(float) * (size_t)p.splits * p.taps * Cout * Cin, 256);
    return PCNN_OK;
}

// x [B,H,W,Cin] bf16, dz [B,H,W,Cout] bf16 -> dW [Cout][ksize*ksize*Cin] f32 = scale * sum_pixels x (*) dz (+ decay * w if w != NULL)
static int wgrad_impl(const void* x_bf16, const void* dz_bf16, int B, int H, int W, int Cin, int Cout, int ksize, float scale,
                      const float* w_f32, float decay, float* dW, void* workspace, size_t workspace_bytes, void* stream, int f16);

extern "C" int pcnn_conv_wgrad_bf16_tc(const void* x_bf16, const void* dz_bf16, int B, int H, int W, int Cin, int Cout, int ksize,
                                       float scale, const float* w_f32, float decay, float* dW, void* workspace, size_t workspace_bytes,
                                       void* stream)
{
    return wgrad_impl(x_bf16, dz_bf16, B, H, W, Cin, Cout, ksize, scale, w_f32, decay, dW, workspace, workspace_bytes, stream, 0);
}

// fully connected layer: x [rows, Cin] fp16, dy [rows, Cout] fp16 -> dW [Cout][Cin] f32 (workspace: pcnn_conv_wgrad_workspace_bytes(1, 1, rows, ...))
extern "C" int pcnn_fc_wgrad_f16_tc(const void* x_f16, const void* dy_f16, int rows, int Cin, int Cout, float scale, const float* w_f32,
                                    float decay, float* dW, void* workspace, size_t workspace_bytes, void* stream)
{
    return wgrad_impl(x_f16, dy_f16, 1, 1, rows, Cin, Cout, 1, scale, w_f32, decay, dW, workspace, workspace_bytes, stream, 1);
}

template <int NB, int F16>
static int launch_wgrad_nb(const CUtensorMap& mx, const CUtensorMap& mz, float* partial, const WgParams& p, int tg_lo, int tg_count,
                           cudaStream_t st)
{
    PCNN_SMEM_OPTIN((k_wgrad_tc<NB, F16>), kWgSmem, "wgrad_tc");
    const unsigned items = (unsigned)((long long)p.splits * tg_count * p.n_tiles * p.m_tiles);
    k_wgrad_tc<NB, F16><<<items, kWgThreads, kWgSmem, st>>>(mx, mz, partial, p, tg_lo, tg_count);
    return check_launch("wgrad_tc");
}

// one launch over tap groups tg_lo .. tg_lo + tg_count - 1, all with nb B blocks per stage (nb = 0 or tg_count = 0: nothing to do)
static int launch_wgrad(int nb, int f16, const CUtensorMap& mx, const CUtensorMap& mz, float* partial, const WgParams& p, int tg_lo,
                        int tg_count, cudaStream_t st)
{
    if (nb == 0 || tg_count == 0) return PCNN_OK;
    PCNN_REQUIRE(nb >= 1 && nb <= kWgMaxNB, "conv_wgrad: %d B blocks per stage", nb);
    switch (nb * 2 + (f16 ? 1 : 0)) {
        case 2: return launch_wgrad_nb<1, 0>(mx, mz, partial, p, tg_lo, tg_count, st);
        case 3: return launch_wgrad_nb<1, 1>(mx, mz, partial, p, tg_lo, tg_count, st);
        case 4: return launch_wgrad_nb<2, 0>(mx, mz, partial, p, tg_lo, tg_count, st);
        case 5: return launch_wgrad_nb<2, 1>(mx, mz, partial, p, tg_lo, tg_count, st);
        case 6: return launch_wgrad_nb<3, 0>(mx, mz, partial, p, tg_lo, tg_count, st);
        case 7: return launch_wgrad_nb<3, 1>(mx, mz, partial, p, tg_lo, tg_count, st);
        case 8: return launch_wgrad_nb<4, 0>(mx, mz, partial, p, tg_lo, tg_count, st);
        default: return launch_wgrad_nb<4, 1>(mx, mz, partial, p, tg_lo, tg_count, st);
    }
}

static int wgrad_impl(const void* x_bf16, const void* dz_bf16, int B, int H, int W, int Cin, int Cout, int ksize, float scale,
                      const float* w_f32, float decay, float* dW, void* workspace, size_t workspace_bytes, void* stream, int f16)
{
    PCNN_REQUIRE(x_bf16 && dz_bf16 && dW && workspace, "conv_wgrad: NULL tensor pointer");
    size_t need = 0;
    int rc = pcnn_conv_wgrad_workspace_bytes(B, H, W, Cin, Cout, ksize, &need);
    if (rc) return rc;
    if (workspace_bytes < need) { set_error("conv_wgrad: workspace too small (%zu < %zu)", workspace_bytes, need); return PCNN_E_WORKSPACE; }
    WgParams p;
    plan(B, H, W, Cin, Cout, ksize, &p);
    p.f16 = f16;
    CUtensorMap mx, mz;
    rc = make_map_nhwc_box(&mx, x_bf16, B, H, W, Cin, p.bw, p.bh);
    if (rc) return rc;
    rc = make_map_nhwc_box(&mz, dz_bf16, B, H, W, Cout, p.bw, p.bh);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const long long items = (long long)p.splits * p.tap_groups * p.n_tiles * p.m_tiles;
    PCNN_REQUIRE(items < 0x7fffffffLL, "conv_wgrad: too many work items");
    if (p.splits == 1) { p.direct = 1; p.scale = scale; p.decay = decay; p.w = w_f32; p.dW = dW; }
    // tap groups of tg taps, then (when tg does not divide the taps) one shorter last group; the paired 64-channel case has
    // two groups of three taps
    const int cb = p.n_tile / 64;
    const int full_groups = p.pair64 ? p.tap_groups : p.taps / p.tg;
    rc = launch_wgrad(full_groups ? p.tg * cb : 0, f16, mx, mz, (float*)workspace, p, 0, full_groups, st);
    if (rc) return rc;
    if (full_groups < p.tap_groups) rc = launch_wgrad((p.taps - full_groups * p.tg) * cb, f16, mx, mz, (float*)workspace, p, full_groups, 1, st);
    if (rc || p.direct) return rc;
    const size_t n4 = (size_t)p.taps * Cout * Cin / 4;
    int blocks = (int)std::min<size_t>((n4 + 255) / 256, (size_t)kNumSMs * 8);
    k_wgrad_finish<<<blocks, 256, 0, st>>>((const float*)workspace, p.splits, p.taps, Cout, Cin, scale, w_f32, decay, dW);
    return check_launch("wgrad_finish");
}

// grid of the element-wise backward kernels: about four CTAs per SM, rounded down to a multiple of cg / gcd(cg, kEwThreads) (cg = C / 8
// channel groups) so that the grid-stride step is a multiple of cg and every thread keeps its channel group (bias_cta_partial)
static int ew_grid(int C)
{
    const int cg = C / 8;
    if (cg < 1) return kNumSMs * 4;
    int a = cg, b = kEwThreads;
    while (b) { const int t = a % b; a = b; b = t; }
    const int q = cg / a;
    return kNumSMs * 4 >= q ? kNumSMs * 4 / q * q : q;
}

// dz = g * [y > 0] (has_relu) or g; optional db [C] = scale * sum_pixels dz (+ decay * b).  bias_ws: >= grid * C floats.
extern "C" int pcnn_relu_bwd_bf16(const void* g_bf16, const void* y_bf16, size_t npix, int C, int has_relu, void* dz_bf16, float scale,
                                  const float* b, float decay, float* db, void* bias_ws, size_t bias_ws_bytes, void* stream)
{
    PCNN_REQUIRE(g_bf16 && (y_bf16 || !has_relu) && (dz_bf16 || db), "relu_bwd: NULL tensor pointer");
    PCNN_REQUIRE(C % 8 == 0 && C >= 8 && C <= 8192, "relu_bwd: C must be a multiple of 8 (got %d)", C);
    const int grid = ew_grid(C);
    PCNN_REQUIRE(!db || (bias_ws && bias_ws_bytes >= sizeof(float) * (size_t)grid * C), "relu_bwd: bias workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    k_relu_bwd<<<grid, kEwThreads, 0, st>>>((const __nv_bfloat16*)g_bf16, (const __nv_bfloat16*)y_bf16, npix, C, has_relu,
                                                                     (__nv_bfloat16*)dz_bf16, db ? (float*)bias_ws : nullptr);
    if (db) k_bias_finish<<<(C + 31) / 32, 256, 0, st>>>((const float*)bias_ws, grid, C, scale, b, decay, db);
    return check_launch("relu_bwd");
}

// max_pool 2x2/2 backward fused with the ReLU mask of the layer below: g [B,H/2,W/2,C], y [B,H,W,C] (pre-pool, post-ReLU) -> dz [B,H,W,C]
extern "C" int pcnn_maxpool_relu_bwd_bf16(const void* g_bf16, const void* y_bf16, int B, int H, int W, int C, void* dz_bf16, float scale,
                                          const float* b, float decay, float* db, void* bias_ws, size_t bias_ws_bytes, void* stream)
{
    PCNN_REQUIRE(g_bf16 && y_bf16 && dz_bf16, "maxpool_relu_bwd: NULL tensor pointer");
    PCNN_REQUIRE(C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "maxpool_relu_bwd: needs even H, W and C %% 8 == 0");
    const int grid = ew_grid(C);
    PCNN_REQUIRE(!db || (bias_ws && bias_ws_bytes >= sizeof(float) * (size_t)grid * C), "maxpool_relu_bwd: bias workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    k_maxpool_relu_bwd<<<grid, kEwThreads, 0, st>>>((const __nv_bfloat16*)g_bf16, (const __nv_bfloat16*)y_bf16, B, H, W, C,
                                                                             (__nv_bfloat16*)dz_bf16, db ? (float*)bias_ws : nullptr);
    if (db) k_bias_finish<<<(C + 31) / 32, 256, 0, st>>>((const float*)bias_ws, grid, C, scale, b, decay, db);
    return check_launch("maxpool_relu_bwd");
}

extern "C" int pcnn_bias_ws_bytes(int C, size_t* bytes)
{
    PCNN_REQUIRE(bytes && C >= 1, "bias_ws_bytes: bad arguments");
    *bytes = sizeof(float) * (size_t)ew_grid(C) * C;
    return PCNN_OK;
}

// out = a + b (+ bf): bf16 tensors a, b (b optional), f32 tensor bf (optional), n elements (multiple of 8)
extern "C" int pcnn_add_to_bf16(const void* a_bf16, const void* b_bf16, const float* b_f32, size_t n, void* out_bf16, void* stream)
{
    PCNN_REQUIRE(a_bf16 && out_bf16 && n % 8 == 0, "add_to_bf16: bad arguments");
    const size_t n8 = n / 8;
    int blocks = (int)std::min<size_t>((n8 + 255) / 256, (size_t)kNumSMs * 8);
    k_add_to_bf16<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)a_bf16, (const __nv_bfloat16*)b_bf16, b_f32, n8,
                                                         (__nv_bfloat16*)out_bf16);
    return check_launch("add_to_bf16");
}
