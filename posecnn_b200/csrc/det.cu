// det.cu — the detection network (lib/networks/vgg16_det.py) from conv_rpn to the fc6 operand, DESIGN.md §16.
//
//   pcnn_rpn_heads_fwd       rpn_cls_score / rpn_bbox_pred (1x1, 512 -> 2A / 4A, both with the ReLU of Network.conv) on the
//                            tensor cores (mma.sync bf16, fp32 accumulation) + the pair softmax of reshape_score /
//                            softmax_high_dimension (channel a against channel A + a); fp32 outputs
//   pcnn_rpn_proposals_fwd   rpn_layer/proposal_layer.py per image: decode + clip, top pre_top_n, bitmask NMS, first post_top_n
//   pcnn_crop_pool_f16       network.py:791-809: crop_and_resize to 14 x 14 + 2 x 2 max-pool -> the fp16 fc6 operand
//   pcnn_softmax_rows_f32    cls_prob = softmax(cls_score) over the classes
//
// Canonical order of the proposals: descending foreground probability, ties by ascending flat anchor index (h, w, a).  The
// reference sorts with numpy's unstable argsort()[::-1] twice (proposal_layer.py and gpu_nms.pyx), so its order among exact
// ties is unspecified; ties are structural here (a pair whose two ReLU'd logits are 0 has probability exactly 0.5).
// All box arithmetic is fp32 in numpy's operation order with every product and sum rounded (no FMA contraction).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "pose_common.cuh"

namespace pcnn {
namespace det {

constexpr int kRpnK = 512;            // conv_rpn channels
constexpr int kRpnPix = 64;           // pixels per CTA: 4 warps x 16 rows
constexpr int kMaxAnchors = 64;
constexpr int kMaxPreTopN = 16384;    // TRAIN.RPN_PRE_NMS_TOP_N is 12000; the sort buffer is 16384 keys (128 KB of shared memory)
constexpr int kSelThreads = 1024;
constexpr int kCrop = 14, kPool = 7;  // crop_and_resize size, then the 2 x 2 / 2 max-pool

__device__ __forceinline__ void mma_bf16_16816(float c[4], const uint32_t a[4], const uint32_t b[2])
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ uint32_t ld_pair(const __nv_bfloat16* p, bool ok)
{
    return ok ? *reinterpret_cast<const uint32_t*>(p) : 0u;
}

// x [npix, 512] bf16, w [6A, 512] bf16 (rows 0..2A-1 rpn_cls_score, 2A..6A-1 rpn_bbox_pred), bias [6A] f32.
// One CTA: 64 pixels x all 6A columns into shared memory, then the epilogue (bias, ReLU, pair softmax) from there.
__global__ void __launch_bounds__(128)
k_rpn_heads(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias, int npix,
            int A, float* __restrict__ cls_prob, float* __restrict__ bbox_pred)
{
    extern __shared__ float acc_s[];   // [kRpnPix][ld]
    const int N = 6 * A, ld = N + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, tig = lane & 3;
    const int p0 = blockIdx.x * kRpnPix;
    const int ra = p0 + warp * 16 + g, rb = ra + 8;
    const __nv_bfloat16* xa = x + (size_t)ra * kRpnK + tig * 2;
    const __nv_bfloat16* xb = x + (size_t)rb * kRpnK + tig * 2;
    const bool oka = ra < npix, okb = rb < npix;
    for (int n0 = 0; n0 < N; n0 += 64) {
        float c[8][4];
#pragma unroll
        for (int t = 0; t < 8; t++) c[t][0] = c[t][1] = c[t][2] = c[t][3] = 0.f;
        for (int k0 = 0; k0 < kRpnK; k0 += 16) {
            uint32_t a[4] = {ld_pair(xa + k0, oka), ld_pair(xb + k0, okb), ld_pair(xa + k0 + 8, oka), ld_pair(xb + k0 + 8, okb)};
#pragma unroll
            for (int t = 0; t < 8; t++) {
                const int n = n0 + t * 8 + g;
                const __nv_bfloat16* wp = w + (size_t)n * kRpnK + k0 + tig * 2;
                uint32_t b[2] = {ld_pair(wp, n < N), ld_pair(wp + 8, n < N)};
                mma_bf16_16816(c[t], a, b);
            }
        }
#pragma unroll
        for (int t = 0; t < 8; t++) {
            const int col = n0 + t * 8 + tig * 2, r = warp * 16 + g;
            if (col < N) { acc_s[r * ld + col] = c[t][0]; acc_s[(r + 8) * ld + col] = c[t][2]; }
            if (col + 1 < N) { acc_s[r * ld + col + 1] = c[t][1]; acc_s[(r + 8) * ld + col + 1] = c[t][3]; }
        }
    }
    __syncthreads();
    // rpn_cls_prob: softmax_high_dimension over the pair (a, A + a) of the ReLU'd scores (network.py:475-488, 700-710)
    for (int i = threadIdx.x; i < kRpnPix * A; i += blockDim.x) {
        const int p = i / A, a = i - p * A, pix = p0 + p;
        if (pix >= npix) continue;
        const float bg = fmaxf(__fadd_rn(acc_s[p * ld + a], bias[a]), 0.f);
        const float fg = fmaxf(__fadd_rn(acc_s[p * ld + A + a], bias[A + a]), 0.f);
        const float m = fmaxf(bg, fg);
        const float e0 = expf(__fsub_rn(bg, m)), e1 = expf(__fsub_rn(fg, m));
        const float s = __fadd_rn(e0, e1);
        cls_prob[(size_t)pix * 2 * A + a] = __fdiv_rn(e0, s);
        cls_prob[(size_t)pix * 2 * A + A + a] = __fdiv_rn(e1, s);
    }
    // rpn_bbox_pred, also ReLU'd (Network.conv's default relu=True)
    for (int i = threadIdx.x; i < kRpnPix * 4 * A; i += blockDim.x) {
        const int p = i / (4 * A), j = i - p * 4 * A, pix = p0 + p;
        if (pix >= npix) continue;
        bbox_pred[(size_t)pix * 4 * A + j] = fmaxf(__fadd_rn(acc_s[p * ld + 2 * A + j], bias[2 * A + j]), 0.f);
    }
}

// ---------------------------------------------------------------------------------------------------- proposals
// 64-bit sort key of anchor i: order-preserving bits of the score above, ~i below (a larger key comes first)
__device__ __forceinline__ uint64_t prop_key(float s, int i)
{
    uint32_t u = __float_as_uint(s);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((uint64_t)u << 32) | (uint32_t)(~(uint32_t)i);
}

// rpn_cls_prob[..., A:] of image b, anchor i = (y * w + x) * A + a
__device__ __forceinline__ float fg_score(const float* cls_prob, size_t img_base, int A, int i)
{
    const int pix = i / A, a = i - pix * A;
    return cls_prob[img_base + (size_t)pix * 2 * A + A + a];
}

// bbox_transform.py:bbox_transform_inv of one box and its deltas (dx, dy, dw, dh), fp32 with every product and sum rounded
__device__ __forceinline__ float4 bbox_transform_inv(const float4 an, const float4 d)
{
    const float wd = __fadd_rn(__fsub_rn(an.z, an.x), 1.f), ht = __fadd_rn(__fsub_rn(an.w, an.y), 1.f);
    const float cx = __fadd_rn(an.x, __fmul_rn(0.5f, wd)), cy = __fadd_rn(an.y, __fmul_rn(0.5f, ht));
    const float pcx = __fadd_rn(__fmul_rn(d.x, wd), cx), pcy = __fadd_rn(__fmul_rn(d.y, ht), cy);
    const float pw = __fmul_rn(expf(d.z), wd), ph = __fmul_rn(expf(d.w), ht);
    const float hw = __fmul_rn(0.5f, pw), hh = __fmul_rn(0.5f, ph);
    return make_float4(__fsub_rn(pcx, hw), __fsub_rn(pcy, hh), __fadd_rn(pcx, hw), __fadd_rn(pcy, hh));
}

// one CTA per image: radix-select the K-th largest key, gather the K keys above it, bitonic-sort them in shared memory,
// decode + clip the sorted boxes (bbox_transform.py:bbox_transform_inv, clip_boxes)
__global__ void __launch_bounds__(kSelThreads)
k_rpn_select(const float* __restrict__ cls_prob, const float* __restrict__ bbox_pred, const float* __restrict__ anchors, int n,
             int A, int K, int sortN, float im_h, float im_w, float4* __restrict__ boxes, float* __restrict__ sorted_scores,
             float* __restrict__ pre_boxes)
{
    extern __shared__ uint64_t skeys[];   // [sortN]
    __shared__ int hist[256];
    __shared__ uint64_t s_prefix, s_mask;
    __shared__ int s_krem, s_count;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31;
    const size_t img_base = (size_t)b * n * 2;   // cls_prob rows of image b: n / A pixels x 2A
    if (t == 0) { s_prefix = 0; s_mask = 0; s_krem = K; s_count = 0; }
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = t; i < 256; i += kSelThreads) hist[i] = 0;
        __syncthreads();
        const uint64_t prefix = s_prefix, mask = s_mask;
        for (int i0 = 0; i0 < n; i0 += kSelThreads) {
            const int i = i0 + t;
            int bin = 256;
            if (i < n) {
                const uint64_t key = prop_key(fg_score(cls_prob, img_base, A, i), i);
                if ((key & mask) == prefix) bin = (int)((key >> shift) & 255);
            }
            const unsigned same = __match_any_sync(0xffffffffu, bin);   // warp-aggregated: scores crowd into a few bins
            if (bin < 256 && lane == __ffs(same) - 1) atomicAdd(&hist[bin], __popc(same));
        }
        __syncthreads();
        if (t == 0) {
            int cum = 0, krem = s_krem, sel = 0;
            for (int d = 255; d >= 0; d--) {
                if (cum + hist[d] >= krem) { sel = d; break; }
                cum += hist[d];
            }
            s_krem = krem - cum;
            s_prefix = prefix | ((uint64_t)sel << shift);
            s_mask = mask | ((uint64_t)255 << shift);
        }
        __syncthreads();
    }
    const uint64_t kth = s_prefix;   // keys are distinct: exactly K keys are >= kth
    for (int i = t; i < n; i += kSelThreads) {
        const uint64_t key = prop_key(fg_score(cls_prob, img_base, A, i), i);
        if (key >= kth) skeys[atomicAdd(&s_count, 1)] = key;
    }
    for (int i = K + t; i < sortN; i += kSelThreads) skeys[i] = 0;
    __syncthreads();
    for (int k = 2; k <= sortN; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = t; i < sortN; i += kSelThreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const uint64_t x = skeys[i], y = skeys[ixj];
                    if (((i & k) == 0) ? (x < y) : (x > y)) { skeys[i] = y; skeys[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
    const float xmax = __fsub_rn(im_w, 1.f), ymax = __fsub_rn(im_h, 1.f);
    for (int r = t; r < K; r += kSelThreads) {
        const int i = (int)(~(uint32_t)skeys[r]);
        const float4 an = reinterpret_cast<const float4*>(anchors)[i];
        const float4 d = reinterpret_cast<const float4*>(bbox_pred)[(size_t)b * n + i];
        float4 o = bbox_transform_inv(an, d);
        o.x = fmaxf(fminf(o.x, xmax), 0.f);
        o.y = fmaxf(fminf(o.y, ymax), 0.f);
        o.z = fmaxf(fminf(o.z, xmax), 0.f);
        o.w = fmaxf(fminf(o.w, ymax), 0.f);
        const float score = fg_score(cls_prob, img_base, A, i);
        boxes[(size_t)b * K + r] = o;
        sorted_scores[(size_t)b * K + r] = score;
        if (pre_boxes) {
            float* q = pre_boxes + ((size_t)b * K + r) * 5;
            q[0] = o.x; q[1] = o.y; q[2] = o.z; q[3] = o.w; q[4] = score;
        }
    }
}

// devIoU of lib/nms/nms_kernel.cu, every operation rounded as numpy's float32 py_cpu_nms does it
__device__ __forceinline__ float dev_iou(const float4 a, const float4 b)
{
    const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    const float width = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
    const float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
    const float inter = __fmul_rn(width, height);
    const float sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.f), __fadd_rn(__fsub_rn(a.w, a.y), 1.f));
    const float sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter));
}

// mask[b][i][cb]: bit j of word cb set when box cb * 64 + j (> i) has IoU > thresh with box i (nms_kernel.cu's layout);
// blocks left of the diagonal are never read by the scan and are not computed
__global__ void __launch_bounds__(64)
k_rpn_nms_mask(const float4* __restrict__ boxes, int K, float thresh, unsigned long long* __restrict__ mask)
{
    const int rb = blockIdx.y, cb = blockIdx.x, b = blockIdx.z, col_blocks = gridDim.x;
    if (cb < rb) return;
    const int row_size = min(K - rb * 64, 64), col_size = min(K - cb * 64, 64);
    __shared__ float4 cols[64];
    const float4* bx = boxes + (size_t)b * K;
    if (threadIdx.x < col_size) cols[threadIdx.x] = bx[cb * 64 + threadIdx.x];
    __syncthreads();
    if (threadIdx.x >= row_size) return;
    const int i = rb * 64 + threadIdx.x;
    const float4 cur = bx[i];
    unsigned long long bits = 0;
    for (int j = (rb == cb ? threadIdx.x + 1 : 0); j < col_size; j++)
        if (dev_iou(cur, cols[j]) > thresh) bits |= 1ull << j;
    mask[((size_t)b * K + i) * col_blocks + cb] = bits;
}

// greedy scan of gpu_nms (nms_kernel.cu:_nms) on one warp per image, stopping at post_top_n kept boxes; writes the capacity
// outputs: kept rows (b, x1, y1, x2, y2) / score, then zero boxes carrying b, and the kept count
__global__ void __launch_bounds__(32)
k_rpn_nms_scan(const float4* __restrict__ boxes, const float* __restrict__ sorted_scores, const unsigned long long* __restrict__ mask,
               int K, int col_blocks, int post_top_n, float* __restrict__ rois, float* __restrict__ scores, int* __restrict__ num_rois)
{
    extern __shared__ unsigned long long remv[];   // [col_blocks]
    const int b = blockIdx.x, lane = threadIdx.x;
    for (int j = lane; j < col_blocks; j += 32) remv[j] = 0;
    const float4* bx = boxes + (size_t)b * K;
    const float* sc = sorted_scores + (size_t)b * K;
    int kept = 0;
    for (int nb = 0; nb < col_blocks && kept < post_top_n; nb++) {
        __syncwarp();
        unsigned long long cur = remv[nb];
        __syncwarp();
        const int end = min(64, K - nb * 64);
        for (int bit = 0; bit < end; bit++) {
            if ((cur >> bit) & 1ull) continue;
            const int i = nb * 64 + bit;
            if (lane < 5) {
                const float4 o = bx[i];
                const float v[5] = {(float)b, o.x, o.y, o.z, o.w};
                rois[((size_t)b * post_top_n + kept) * 5 + lane] = v[lane];
                if (lane == 0) scores[(size_t)b * post_top_n + kept] = sc[i];
            }
            if (++kept == post_top_n) break;
            const unsigned long long* row = mask + ((size_t)b * K + i) * col_blocks;
            cur |= row[nb];
            for (int j = nb + 1 + lane; j < col_blocks; j += 32) remv[j] |= row[j];
        }
    }
    for (int r = kept + lane; r < post_top_n; r += 32) {
        float* q = rois + ((size_t)b * post_top_n + r) * 5;
        q[0] = (float)b; q[1] = q[2] = q[3] = q[4] = 0.f;
        scores[(size_t)b * post_top_n + r] = 0.f;
    }
    if (lane == 0) num_rois[b] = kept;
}

// ---------------------------------------------------------------------------------------------------- crop pool
// crop_and_resize (TF 1.x, bilinear, extrapolation 0) of box (x1, y1, x2, y2) / ((W - 1) * stride, (H - 1) * stride) to 14 x 14,
// then max_pool2d 2 x 2 / 2 'SAME' -> [N, 7, 7, C] fp16 (saturated to +-65504).  One CTA per (roi, pooled row); a thread owns
// eight channels of one pooled cell.
__device__ __forceinline__ void bf16x8_to_f32(const uint4 v, float f[8])
{
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int k = 0; k < 4; k++) { const float2 p = __bfloat1622float2(h[k]); f[2 * k] = p.x; f[2 * k + 1] = p.y; }
}

__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), t)); }

__global__ void __launch_bounds__(256)
k_crop_pool(const __nv_bfloat16* __restrict__ feat, int B, int H, int W, int C, const float* __restrict__ rois, int roi_stride,
            float feat_stride, __half* __restrict__ out)
{
    const int r = blockIdx.x, ph = blockIdx.y, cg = C / 8;
    const float* roi = rois + (size_t)r * roi_stride;
    const int b = (int)roi[0];
    const float hn = __fmul_rn((float)(H - 1), feat_stride), wn = __fmul_rn((float)(W - 1), feat_stride);
    const float x1 = __fdiv_rn(roi[1], wn), y1 = __fdiv_rn(roi[2], hn), x2 = __fdiv_rn(roi[3], wn), y2 = __fdiv_rn(roi[4], hn);
    const float hm1 = (float)(H - 1), wm1 = (float)(W - 1);
    const float hs = __fdiv_rn(__fmul_rn(__fsub_rn(y2, y1), hm1), (float)(kCrop - 1));
    const float ws = __fdiv_rn(__fmul_rn(__fsub_rn(x2, x1), wm1), (float)(kCrop - 1));
    const bool valid_b = b >= 0 && b < B;
    for (int item = threadIdx.x; item < kPool * cg; item += blockDim.x) {
        const int pw = item / cg, c0 = (item - pw * cg) * 8;
        float best[8];
#pragma unroll
        for (int k = 0; k < 8; k++) best[k] = -INFINITY;
#pragma unroll
        for (int dy = 0; dy < 2; dy++) {
            const float in_y = __fadd_rn(__fmul_rn(y1, hm1), __fmul_rn((float)(2 * ph + dy), hs));
            const bool oky = valid_b && !(in_y < 0.f || in_y > hm1);
            const int ty = oky ? (int)floorf(in_y) : 0, by = oky ? (int)ceilf(in_y) : 0;
            const float yl = __fsub_rn(in_y, (float)ty);
#pragma unroll
            for (int dx = 0; dx < 2; dx++) {
                const float in_x = __fadd_rn(__fmul_rn(x1, wm1), __fmul_rn((float)(2 * pw + dx), ws));
                float v[8];
                if (oky && !(in_x < 0.f || in_x > wm1)) {
                    const int lx = (int)floorf(in_x), rx = (int)ceilf(in_x);
                    const float xl = __fsub_rn(in_x, (float)lx);
                    const __nv_bfloat16* base = feat + (size_t)b * H * W * C + c0;
                    float tl[8], tr[8], bl[8], br[8];
                    bf16x8_to_f32(*reinterpret_cast<const uint4*>(base + ((size_t)ty * W + lx) * C), tl);
                    bf16x8_to_f32(*reinterpret_cast<const uint4*>(base + ((size_t)ty * W + rx) * C), tr);
                    bf16x8_to_f32(*reinterpret_cast<const uint4*>(base + ((size_t)by * W + lx) * C), bl);
                    bf16x8_to_f32(*reinterpret_cast<const uint4*>(base + ((size_t)by * W + rx) * C), br);
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const float top = lerp_rn(tl[k], tr[k], xl), bot = lerp_rn(bl[k], br[k], xl);
                        v[k] = lerp_rn(top, bot, yl);
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < 8; k++) v[k] = 0.f;
                }
#pragma unroll
                for (int k = 0; k < 8; k++) best[k] = fmaxf(best[k], v[k]);
            }
        }
        __align__(16) __half o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) o[k] = __float2half_rn(sat_f16(best[k]));
        *reinterpret_cast<uint4*>(out + ((size_t)r * kPool * kPool + ph * kPool + pw) * C + c0) = *reinterpret_cast<const uint4*>(o);
    }
}

// softmax over a row (tf.nn.softmax): one warp per row
__global__ void __launch_bounds__(256)
k_softmax_rows(const float* __restrict__ in, int rows, int cols, float* __restrict__ out)
{
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* x = in + (size_t)row * cols;
    float m = -INFINITY;
    for (int j = lane; j < cols; j += 32) m = fmaxf(m, x[j]);
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < cols; j += 32) s += expf(x[j] - m);
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int j = lane; j < cols; j += 32) out[(size_t)row * cols + j] = expf(x[j] - m) / s;
}

// ---------------------------------------------------------------------------------------------------- detection records
// lib/fcn/test.py's post-processing of the detection network (1589-1616, 1639-1691, 1731-1746) for one (image, class j >= 1) slot
// per CTA: the argmax of cls_prob[:, j] over the kept proposals above 0.02, its de-normalised and clipped class-j box, and the
// depth z of compute_translations' Nelder-Mead fit (scipy 1.18.1 _minimize_neldermead at N = 1).  Every thread runs the same
// scalar Nelder-Mead decisions on the objective values the block computes together, so control flow stays uniform.
constexpr int kRecThreads = 256;
constexpr int kRecMaxPoints = 4096;
constexpr int kRecMaxClasses = 128;
constexpr int kNmMaxFun = 200;   // maxiter = maxfun = 200 * N

// np.minimum / np.maximum: NaN propagates (fminf / fmaxf would drop it)
__device__ __forceinline__ double nan_min(double a, double b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }
// clip_boxes: np.maximum(np.minimum(v, hi), 0) with numpy's scalar rules (NaN kept, ties keep the first operand)
__device__ __forceinline__ float clip_f(float v, float hi)
{
    const float m = (v <= hi || v != v) ? v : hi;
    return (m >= 0.f || m != m) ? m : 0.f;
}

// np.argsort of two values (insertion sort: stable, NaN last): true when the second sorts before the first
__device__ __forceinline__ bool nm_swap(double f0, double f1) { return f1 < f0 || (f0 != f0 && f1 == f1); }

struct RecObjective {
    const float* pts;   // [P,3] of the slot's class, in shared memory
    int P;
    float R[9];
    double K[9], rx, ry, width, height;
    double (*red)[kRecThreads / 32][4];   // [2][warps][xmin, xmax, ymin, ymax]
};

// distance_objective(z): fp32 camera coordinates ((r0 px + r1 py) + r2 pz) + t with t = f32(rx z, ry z, z), the K row products
// and the division in fp64, NaN-propagating extents, (w - width)^2 + (h - height)^2.  Called by every thread of the block.
__device__ __forceinline__ double rec_objective(const RecObjective& o, double z, int& parity)
{
    const float t[3] = {(float)__dmul_rn(o.rx, z), (float)__dmul_rn(o.ry, z), (float)z};
    double x1 = INFINITY, x2 = -INFINITY, y1 = INFINITY, y2 = -INFINITY;
    for (int p = threadIdx.x; p < o.P; p += kRecThreads) {
        const float px = o.pts[3 * p], py = o.pts[3 * p + 1], pz = o.pts[3 * p + 2];
        double c[3];
#pragma unroll
        for (int r = 0; r < 3; r++)
            c[r] = (double)__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(o.R[3 * r], px), __fmul_rn(o.R[3 * r + 1], py)),
                                               __fmul_rn(o.R[3 * r + 2], pz)), t[r]);
        double q[3];
#pragma unroll
        for (int r = 0; r < 3; r++)
            q[r] = __dadd_rn(__dadd_rn(__dmul_rn(o.K[3 * r], c[0]), __dmul_rn(o.K[3 * r + 1], c[1])), __dmul_rn(o.K[3 * r + 2], c[2]));
        const double u = __ddiv_rn(q[0], q[2]), v = __ddiv_rn(q[1], q[2]);
        x1 = nan_min(x1, u); x2 = nan_max(x2, u); y1 = nan_min(y1, v); y2 = nan_max(y2, v);
    }
    for (int off = 16; off; off >>= 1) {
        x1 = nan_min(x1, __shfl_xor_sync(0xffffffffu, x1, off)); x2 = nan_max(x2, __shfl_xor_sync(0xffffffffu, x2, off));
        y1 = nan_min(y1, __shfl_xor_sync(0xffffffffu, y1, off)); y2 = nan_max(y2, __shfl_xor_sync(0xffffffffu, y2, off));
    }
    double (*red)[4] = o.red[parity];
    parity ^= 1;   // alternate buffers: one barrier per evaluation
    if ((threadIdx.x & 31) == 0) {
        double* r = red[threadIdx.x >> 5];
        r[0] = x1; r[1] = x2; r[2] = y1; r[3] = y2;
    }
    __syncthreads();
    x1 = red[0][0]; x2 = red[0][1]; y1 = red[0][2]; y2 = red[0][3];
    for (int w = 1; w < kRecThreads / 32; w++) {
        x1 = nan_min(x1, red[w][0]); x2 = nan_max(x2, red[w][1]); y1 = nan_min(y1, red[w][2]); y2 = nan_max(y2, red[w][3]);
    }
    const double dw = __dsub_rn(__dsub_rn(x2, x1), o.width), dh = __dsub_rn(__dsub_rn(y2, y1), o.height);
    return __dadd_rn(__dmul_rn(dw, dw), __dmul_rn(dh, dh));
}

// _wrap_scalar_function_maxfun_validation: the 201st call raises _MaxFuncCallError instead of evaluating
__device__ __forceinline__ bool nm_call(const RecObjective& o, double x, double& fx, int& nfev, int& parity)
{
    if (nfev >= kNmMaxFun) return false;
    nfev++;
    fx = rec_objective(o, x, parity);
    return true;
}

// scipy.optimize._optimize._minimize_neldermead at N = 1, x0 = 0.5, defaults (rho 1, chi 2, psi 0.5, sigma 0.5, xatol = fatol =
// 1e-4, maxiter = maxfun = 200), with its expression shapes.  For N = 1 xbar = sim[0] and fsim[-2] = fsim[0], so the
// reflection's `fxr < fsim[-2]` branch can never be taken after `fxr < fsim[0]` failed.  Returns sim[0].
__device__ __forceinline__ double nelder_mead(const RecObjective& o, int& nit, int& nfev)
{
    int parity = 0;
    nfev = 0;
    double s0 = 0.5, s1 = __dmul_rn(__dadd_rn(1.0, 0.05), 0.5), f0, f1;   // sim[1] = (1 + nonzdelt) * x0
    nm_call(o, s0, f0, nfev, parity);
    nm_call(o, s1, f1, nfev, parity);
    if (nm_swap(f0, f1)) { const double ts = s0, tf = f0; s0 = s1; f0 = f1; s1 = ts; f1 = tf; }
    int it = 1;
    while (nfev < kNmMaxFun && it < kNmMaxFun) {
        if (fabs(__dsub_rn(s1, s0)) <= 1e-4 && fabs(__dsub_rn(f0, f1)) <= 1e-4) break;
        do {   // `break` below is scipy's `except _MaxFuncCallError: pass`
            const double xbar = s0;
            const double xr = __dsub_rn(__dmul_rn(2.0, xbar), __dmul_rn(1.0, s1));
            double fxr;
            if (!nm_call(o, xr, fxr, nfev, parity)) break;
            if (fxr < f0) {
                const double xe = __dsub_rn(__dmul_rn(3.0, xbar), __dmul_rn(2.0, s1));
                double fxe;
                if (!nm_call(o, xe, fxe, nfev, parity)) break;
                if (fxe < fxr) { s1 = xe; f1 = fxe; } else { s1 = xr; f1 = fxr; }
            } else {
                bool shrink = false;
                if (fxr < f1) {
                    const double xc = __dsub_rn(__dmul_rn(1.5, xbar), __dmul_rn(0.5, s1));
                    double fxc;
                    if (!nm_call(o, xc, fxc, nfev, parity)) break;
                    if (fxc <= fxr) { s1 = xc; f1 = fxc; } else shrink = true;
                } else {
                    const double xcc = __dadd_rn(__dmul_rn(0.5, xbar), __dmul_rn(0.5, s1));
                    double fxcc;
                    if (!nm_call(o, xcc, fxcc, nfev, parity)) break;
                    if (fxcc < f1) { s1 = xcc; f1 = fxcc; } else shrink = true;
                }
                if (shrink) {
                    s1 = __dadd_rn(s0, __dmul_rn(0.5, __dsub_rn(s1, s0)));
                    double fs;
                    if (!nm_call(o, s1, fs, nfev, parity)) break;
                    f1 = fs;
                }
            }
            it++;
        } while (false);
        if (nm_swap(f0, f1)) { const double ts = s0, tf = f0; s0 = s1; f0 = f1; s1 = ts; f1 = tf; }
    }
    nit = it;
    return s0;
}

struct RecArgs {
    const float *cls_prob, *bbox_pred, *poses_tanh, *rois;
    const int32_t* num_rois;
    int rows, C, P, num_meta;
    float xmax, ymax;
    const float *meta, *points;
    float *dets, *poses;
    int32_t *num_dets, *trace;
};

__global__ void __launch_bounds__(kRecThreads) k_det_records(RecArgs a)
{
    extern __shared__ float s_pts[];   // [P,3]
    __shared__ double s_red[2][kRecThreads / 32][4];
    __shared__ unsigned long long s_best[kRecThreads / 32];
    const int j = blockIdx.x + 1, b = blockIdx.y, C = a.C, t = threadIdx.x, lane = t & 31;
    const size_t slot = (size_t)b * (C - 1) + (j - 1);
    const int nr = min(max(a.num_rois[b], 0), a.rows);
    // argmax over rows r < nr with score > 0.02f; key = (score bits, ~r): the largest key is the top score at the lowest row.
    // Scores above 0.02 are positive, so their bit patterns order as the values; NaN fails the comparison.
    unsigned long long best = 0;
    for (int r = t; r < nr; r += kRecThreads) {
        const float s = a.cls_prob[((size_t)b * a.rows + r) * C + j];
        if (s > 0.02f) {
            const unsigned long long key = ((unsigned long long)__float_as_uint(s) << 32) | (uint32_t)~(uint32_t)r;
            best = key > best ? key : best;
        }
    }
    for (int off = 16; off; off >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, off);
        best = o > best ? o : best;
    }
    if (lane == 0) s_best[t >> 5] = best;
    for (int p = t; p < a.P * 3; p += kRecThreads) s_pts[p] = a.points[(size_t)j * a.P * 3 + p];
    __syncthreads();
    best = s_best[0];
    for (int w = 1; w < kRecThreads / 32; w++) best = s_best[w] > best ? s_best[w] : best;
    float* det = a.dets + slot * 7;
    float* pose = a.poses + slot * 7;
    int32_t* tr = a.trace + slot * 2;
    if (best == 0) {   // nothing above the threshold: an empty slot
        if (t < 7) { det[t] = t == 0 ? (float)b : 0.f; pose[t] = 0.f; }
        if (t < 2) tr[t] = 0;
        return;
    }
    const int r = (int)~(uint32_t)best;
    const size_t row = (size_t)b * a.rows + r;
    const float* q = a.poses_tanh + row * 4 * C + 4 * j;
    __shared__ float s_box[4], s_R[9];
    __shared__ double s_ray[4];   // rx, ry, width, height
    if (t == 0) {
        // test.py:1731-1743: bbox_pred *= stds (float64, stored back to float32), += means (0); boxes = rois[:, 1:5] / im_scale (1)
        const float* dp = a.bbox_pred + row * 4 * C + 4 * j;
        const double stds[4] = {0.1, 0.1, 0.2, 0.2};
        float dn[4];
#pragma unroll
        for (int k = 0; k < 4; k++) dn[k] = (float)__dadd_rn((double)(float)__dmul_rn((double)dp[k], stds[k]), 0.0);
        const float* roi = a.rois + row * 5;
        float4 box = bbox_transform_inv(make_float4(roi[1], roi[2], roi[3], roi[4]), make_float4(dn[0], dn[1], dn[2], dn[3]));
        box.x = clip_f(box.x, a.xmax); box.y = clip_f(box.y, a.ymax); box.z = clip_f(box.z, a.xmax); box.w = clip_f(box.w, a.ymax);
        s_box[0] = box.x; s_box[1] = box.y; s_box[2] = box.z; s_box[3] = box.w;
        // compute_translations (test.py:1646-1653): centre and size in float32 (x * 0.5f is x / 2 exactly), the ray in float64
        const float* m = a.meta + (size_t)b * a.num_meta;
        const float cxf = __fmul_rn(__fadd_rn(box.x, box.z), 0.5f), cyf = __fmul_rn(__fadd_rn(box.y, box.w), 0.5f);
        s_ray[0] = __ddiv_rn(__dsub_rn((double)cxf, (double)m[2]), (double)m[0]);
        s_ray[1] = __ddiv_rn(__dsub_rn((double)cyf, (double)m[5]), (double)m[4]);
        s_ray[2] = (double)__fsub_rn(box.z, box.x);
        s_ray[3] = (double)__fsub_rn(box.w, box.y);
        quat2mat_f32(q[0], q[1], q[2], q[3], s_R);
    }
    __syncthreads();
    RecObjective o;
    o.pts = s_pts;
    o.P = a.P;
    o.red = s_red;
    const float* m = a.meta + (size_t)b * a.num_meta;
#pragma unroll
    for (int k = 0; k < 9; k++) { o.K[k] = (double)m[k]; o.R[k] = s_R[k]; }
    o.rx = s_ray[0]; o.ry = s_ray[1]; o.width = s_ray[2]; o.height = s_ray[3];
    int nit, nfev;
    const double z = nelder_mead(o, nit, nfev);
    if (t == 0) {
        const float d[7] = {(float)b, (float)j, s_box[0], s_box[1], s_box[2], s_box[3], __uint_as_float((uint32_t)(best >> 32))};
        const float p[7] = {q[0], q[1], q[2], q[3], (float)__dmul_rn(o.rx, z), (float)__dmul_rn(o.ry, z), (float)z};
#pragma unroll
        for (int k = 0; k < 7; k++) { det[k] = d[k]; pose[k] = p[k]; }
        tr[0] = nit;
        tr[1] = nfev;
        atomicAdd(a.num_dets + b, 1);
    }
}

struct PropLayout {
    int K, sortN, col_blocks;
    size_t boxes, scores, mask, total;
};

static int prop_layout(int B, int h, int w, int A, int pre_top_n, PropLayout* L)
{
    PCNN_REQUIRE(B >= 1 && B <= 65535 && h >= 1 && w >= 1 && A >= 1, "rpn_proposals: non-positive size (B %d, h %d, w %d, A %d)",
                 B, h, w, A);
    PCNN_REQUIRE(A <= kMaxAnchors, "rpn_proposals: A = %d anchors per position (at most %d)", A, kMaxAnchors);
    PCNN_REQUIRE((long long)h * w * A <= (1 << 30), "rpn_proposals: %d x %d x %d anchors", h, w, A);
    PCNN_REQUIRE(pre_top_n >= 1 && pre_top_n <= kMaxPreTopN, "rpn_proposals: pre_top_n %d outside [1, %d]", pre_top_n,
                 kMaxPreTopN);
    const int n = h * w * A;
    L->K = pre_top_n < n ? pre_top_n : n;   // proposal_layer.py: order[:pre_nms_topN]
    L->sortN = 1;
    while (L->sortN < L->K) L->sortN <<= 1;
    L->col_blocks = (L->K + 63) / 64;
    size_t off = 0;
    L->boxes = off; off = align_up(off + sizeof(float4) * (size_t)B * L->K, 256);
    L->scores = off; off = align_up(off + sizeof(float) * (size_t)B * L->K, 256);
    L->mask = off; off = align_up(off + sizeof(unsigned long long) * (size_t)B * L->K * L->col_blocks, 256);
    L->total = off;
    return PCNN_OK;
}

}  // namespace det
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::det;

extern "C" int pcnn_rpn_heads_fwd(const void* conv_rpn_bf16, const void* weights_bf16, const float* bias, int npix, int A,
                                  float* cls_prob, float* bbox_pred, void* stream)
{
    PCNN_REQUIRE(conv_rpn_bf16 && weights_bf16 && bias && cls_prob && bbox_pred, "rpn_heads: NULL tensor pointer");
    PCNN_REQUIRE(npix >= 1 && A >= 1, "rpn_heads: non-positive size (npix %d, A %d)", npix, A);
    PCNN_REQUIRE(A <= kMaxAnchors, "rpn_heads: A = %d anchors per position (at most %d)", A, kMaxAnchors);
    const size_t smem = sizeof(float) * kRpnPix * (6 * A + 1);
    PCNN_SMEM_OPTIN(k_rpn_heads, sizeof(float) * kRpnPix * (6 * kMaxAnchors + 1), "rpn_heads");
    const int grid = (npix + kRpnPix - 1) / kRpnPix;
    k_rpn_heads<<<grid, 128, smem, (cudaStream_t)stream>>>((const __nv_bfloat16*)conv_rpn_bf16, (const __nv_bfloat16*)weights_bf16,
                                                          bias, npix, A, cls_prob, bbox_pred);
    return check_launch("rpn_heads");
}

extern "C" int pcnn_rpn_proposals_workspace_bytes(int B, int h, int w, int A, int pre_top_n, size_t* bytes)
{
    PCNN_REQUIRE(bytes, "rpn_proposals: NULL bytes");
    PropLayout L;
    const int rc = prop_layout(B, h, w, A, pre_top_n, &L);
    if (rc) return rc;
    *bytes = L.total;
    return PCNN_OK;
}

extern "C" int pcnn_rpn_proposals_fwd(const float* cls_prob, const float* bbox_pred, const float* anchors, int B, int h, int w, int A,
                                      float im_h, float im_w, int pre_top_n, int post_top_n, float nms_thresh, float* rois,
                                      float* scores, int32_t* num_rois, float* pre_boxes, void* workspace, size_t workspace_bytes,
                                      void* stream)
{
    PCNN_REQUIRE(cls_prob && bbox_pred && anchors && rois && scores && num_rois && workspace, "rpn_proposals: NULL tensor pointer");
    PropLayout L;
    int rc = prop_layout(B, h, w, A, pre_top_n, &L);
    if (rc) return rc;
    PCNN_REQUIRE(post_top_n >= 1, "rpn_proposals: post_top_n %d < 1", post_top_n);
    PCNN_REQUIRE(im_h >= 1.f && im_w >= 1.f, "rpn_proposals: image size %g x %g", im_h, im_w);
    if (workspace_bytes < L.total) {
        set_error("rpn_proposals: workspace too small (%zu < %zu)", workspace_bytes, L.total);
        return PCNN_E_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    float4* boxes = (float4*)(ws + L.boxes);
    float* sorted_scores = (float*)(ws + L.scores);
    unsigned long long* mask = (unsigned long long*)(ws + L.mask);
    const int n = h * w * A;
    const size_t sel_smem = sizeof(uint64_t) * L.sortN;
    PCNN_SMEM_OPTIN(k_rpn_select, sizeof(uint64_t) * kMaxPreTopN, "rpn_select");
    k_rpn_select<<<B, kSelThreads, sel_smem, st>>>(cls_prob, bbox_pred, anchors, n, A, L.K, L.sortN, im_h, im_w, boxes, sorted_scores,
                                                   pre_boxes);
    rc = check_launch("rpn_select");
    if (rc) return rc;
    dim3 grid(L.col_blocks, L.col_blocks, B);
    k_rpn_nms_mask<<<grid, 64, 0, st>>>(boxes, L.K, nms_thresh, mask);
    rc = check_launch("rpn_nms_mask");
    if (rc) return rc;
    k_rpn_nms_scan<<<B, 32, sizeof(unsigned long long) * L.col_blocks, st>>>(boxes, sorted_scores, mask, L.K, L.col_blocks,
                                                                             post_top_n, rois, scores, num_rois);
    return check_launch("rpn_nms_scan");
}

extern "C" int pcnn_crop_pool_f16(const void* feat_bf16, int B, int H, int W, int C, const float* rois, int num_rois, int roi_stride,
                                  float feat_stride, void* out_f16, void* stream)
{
    PCNN_REQUIRE(feat_bf16 && rois && out_f16, "crop_pool: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 2 && W >= 2 && num_rois >= 1 && roi_stride >= 5 && feat_stride > 0.f,
                 "crop_pool: bad shape (B %d, H %d, W %d, rois %d x %d)", B, H, W, num_rois, roi_stride);
    PCNN_REQUIRE(C >= 8 && C % 8 == 0, "crop_pool: C = %d must be a positive multiple of 8", C);
    PCNN_REQUIRE(num_rois <= 0x7fffffff / kPool, "crop_pool: %d rois", num_rois);
    dim3 grid(num_rois, kPool);
    k_crop_pool<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)feat_bf16, B, H, W, C, rois, roi_stride, feat_stride,
                                                        (__half*)out_f16);
    return check_launch("crop_pool");
}

extern "C" int pcnn_softmax_rows_f32(const float* in, int rows, int cols, float* out, void* stream)
{
    PCNN_REQUIRE(in && out, "softmax_rows: NULL tensor pointer");
    PCNN_REQUIRE(rows >= 1 && cols >= 1, "softmax_rows: non-positive size (%d x %d)", rows, cols);
    k_softmax_rows<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(in, rows, cols, out);
    return check_launch("softmax_rows");
}

extern "C" int pcnn_det_records_fwd(const float* cls_prob, const float* bbox_pred, const float* poses_tanh, const float* rois,
                                    const int32_t* num_rois, int B, int rows, int C, int im_h, int im_w, const float* meta,
                                    int num_meta, const float* points, int P, float* dets, float* poses, int32_t* num_dets,
                                    int32_t* trace, void* stream)
{
    PCNN_REQUIRE(cls_prob && bbox_pred && poses_tanh && rois && num_rois && meta && points && dets && poses && num_dets && trace,
                 "det_records: NULL tensor pointer");
    PCNN_REQUIRE(C >= 2 && C <= kRecMaxClasses, "det_records: C = %d classes (2 <= C <= %d)", C, kRecMaxClasses);
    PCNN_REQUIRE(P >= 1 && P <= kRecMaxPoints, "det_records: P = %d points per class (1 <= P <= %d)", P, kRecMaxPoints);
    PCNN_REQUIRE(B >= 1 && B <= 65535, "det_records: B = %d images (1 <= B <= 65535)", B);
    PCNN_REQUIRE(rows >= 1 && (long long)B * rows * 4 * C <= 0x7fffffffLL, "det_records: %d rows per image", rows);
    PCNN_REQUIRE(im_h >= 1 && im_w >= 1, "det_records: image size %d x %d", im_h, im_w);
    PCNN_REQUIRE(num_meta >= 9, "det_records: num_meta = %d (K is meta[b, 0:9])", num_meta);
    cudaStream_t st = (cudaStream_t)stream;
    const cudaError_t e = cudaMemsetAsync(num_dets, 0, sizeof(int32_t) * B, st);
    if (e != cudaSuccess) {
        set_error("det_records: %s", cudaGetErrorString(e));
        return PCNN_E_CUDA;
    }
    RecArgs a{cls_prob, bbox_pred, poses_tanh, rois, num_rois, rows, C, P, num_meta, (float)(im_w - 1), (float)(im_h - 1), meta, points,
              dets, poses, num_dets, trace};
    PCNN_SMEM_OPTIN(k_det_records, sizeof(float) * 3 * kRecMaxPoints, "det_records");
    k_det_records<<<dim3(C - 1, B), kRecThreads, sizeof(float) * 3 * P, st>>>(a);
    return check_launch("det_records");
}
