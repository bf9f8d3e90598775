// hough_vote.cu — Houghvotinggpu for sm_90a, whole batch per call, no host round trips.
//
// Behavioural spec: lib/hough_voting_gpu_layer/hough_voting_gpu_op.cu.cc:253-333 (vote
// predicate: cosine cone > inlier, clipped to a depth-dependent square), :335-383 (maxima),
// :386-576 (ROI / pose rows), hough_voting_gpu_op.cc:321-428 (batch loop, MAX_ROI/B cap,
// dummy row).  See DESIGN.md §3 for the algorithm; in short:
//
//   The reference evaluates the predicate for every (cell, sampled pixel) pair — a gather of
//   count*H*W*(N/skip) cosine tests.  Here each sampled pixel scatters its vote set instead.
//   On one image row the vote set of a pixel is (cone ∩ row ∩ square) = ONE interval of
//   cells, so a pixel contributes "+1 at the first cell, -1 after the last cell" to a
//   per-row difference array, and an inclusive prefix sum along the row yields exactly the
//   vote counts.  Interval end points are estimated analytically (two boundary rays) and
//   then snapped with the reference's own fp32 predicate, so the result equals the per-cell
//   evaluation wherever that predicate is monotone along the row (everywhere outside
//   rounding distance of the threshold).
//
//   k_hist     per-chunk class histogram and class totals (+ zero-fill of the output buffers)
//   k_emit     class filter (> label_threshold), deterministic raster-order ranks; every skip-th
//              pixel of a class becomes a 32-byte sample record (direction, depth, window,
//              boundary-ray slopes); records are built on densely packed lanes from a smem queue
//   k_worklist (image, class, 16-row band) work items inside each class's vote bounding box,
//              heaviest classes first
//   k_vote     persistent CTAs: difference array of a band in shared memory, shared-memory
//              atomics (2 per sample-row), row prefix scan fused with the arg-max; end points
//              that fall within rounding distance of a cell are queued per warp and re-checked
//              with the reference predicate on densely packed lanes
//   k_select / k_localmax   maxima (first arg-max per class, or 7x7 local maxima)
//   k_celldata per selected cell: exact recount, mean depth, box extents (second pass of the
//              reference kernel, done only for selected cells)
//   k_finalize ROI cap, row offsets, ROI / pose / target / weight / domain rows
#include <float.h>
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "heads_common.cuh"

namespace pcnn {
namespace hough {

constexpr int kChunk = 2048;      // pixels per CTA in k_hist / k_emit
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kCandCapThr = 4096; // candidate capacity per image in threshold mode
constexpr int kMaxM = 16383;

struct __align__(16) Sample {
    int xy;       // x | y << 16
    float u, v;   // predicted direction (vertex channels 3c, 3c+1)
    float n1;     // |(u,v)| rounded like the reference (angle_distance, .cu.cc:36)
    float k1, k2; // dx = dy * k for the two boundary rays of the cone
    int mflags;   // window half-size m (cells with |dx|,|dy| <= m pass `< threshold`) | flags << 16
    float d;      // exp(vertex channel 3c+2)
};
static_assert(sizeof(Sample) == 32, "sample record is two 16-byte vectors");

// Where k_emit gets a sampled pixel's (u, v, log z): the dense vertex_pred tensor [B,H,W,3C] (the op's registered
// input, hough_voting_gpu_op.cc:37-52), or — inside the network pipeline — the 1/8-resolution head tensor
// `lowres` [B,H/8,W/8,4C] (channels C.. = vertex head before the x8 bilinear up-sampling) + the vertex_pred bias:
// the three values are then computed on demand with k_up8_heads' own operation sequence (heads_common.cuh), so the
// 2.6 GB dense tensor (batch 32) is never written.  Bit-identical results (tests/test_network_gpu.py).
struct VertexSrc {
    const float* dense;
    const float* lowres;
    const float* bias;
    int h, w;   // low-resolution size (H / 8, W / 8)
};

struct Layout {
    int nchunks, nbands, R, samp_cap, cand_cap;
    size_t chunk_hist, cls_size, cls_slot, cls_nsamp, cls_soff, slot_cls, img_count, bbox, samples, band_res, work,
        work_ctr, cand_key, cand_val, cand_n, cand_data, votes, total;
};

static int band_rows(int B, int H, int W, int C)
{
    // difference array of one band: R rows x (W + 3) ints; 16 rows = 41 KB at W = 640, so four
    // CTAs (32 warps) fit per SM and the work items are fine grained enough to balance
    int R = 16;
    while (R > 1 && (size_t)R * (W + 3) * 4 > 48 * 1024) R >>= 1;
    // Small batches (an image shard of a multi-GPU batch, configs[1]): an item's cost is its class's samples x R rows and the kernel
    // cannot finish before its heaviest item, so with few items (B x C x H / R < ~16 per resident CTA) the bands are halved:
    // measured (profiles/r02_hough_band_rows_sweep.txt) batch 1: 0.087 -> 0.071 ms, batch 4: 0.194 -> 0.136 ms on the 8(d) scenes,
    // 0.39 -> 0.24 ms on the network's maps; 4 and 2 rows bring nothing more.  Results do not depend on R (tests run B = 1, 2, 4
    // and 32).  PCNN_HOUGH_BAND_ROWS overrides (power of two).
    static const int forced = getenv("PCNN_HOUGH_BAND_ROWS") ? atoi(getenv("PCNN_HOUGH_BAND_ROWS")) : 0;
    if (forced >= 1 && forced <= R && (forced & (forced - 1)) == 0) return forced;
    static const int min_rows = getenv("PCNN_HOUGH_BAND_MIN") ? atoi(getenv("PCNN_HOUGH_BAND_MIN")) : 8;
    const long long want = 16LL * 4 * kNumSMs;
    while (R > min_rows && (long long)B * C * ((H + R - 1) / R) < want) R >>= 1;
    return R;
}

static Layout make_layout(int B, int H, int W, int C, int skip, bool want_votes, bool threshold_mode)
{
    Layout L;
    size_t HW = (size_t)H * W;
    L.nchunks = (int)((HW + kChunk - 1) / kChunk);
    L.R = band_rows(B, H, W, C);
    L.nbands = (H + L.R - 1) / L.R;
    L.samp_cap = (int)((HW + skip - 1) / skip) + C;
    L.cand_cap = threshold_mode ? kCandCapThr : C;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.chunk_hist = take(sizeof(int) * (size_t)B * L.nchunks * C);
    L.cls_size = take(sizeof(int) * (size_t)B * C);
    L.cls_slot = take(sizeof(int) * (size_t)B * C);
    L.cls_nsamp = take(sizeof(int) * (size_t)B * C);
    L.cls_soff = take(sizeof(int) * (size_t)B * C);
    L.slot_cls = take(sizeof(int) * (size_t)B * C);
    L.img_count = take(sizeof(int) * (size_t)B);
    L.bbox = take(sizeof(int) * (size_t)B * C * 4);
    L.samples = take(sizeof(Sample) * (size_t)B * L.samp_cap);
    L.band_res = take(sizeof(int2) * (size_t)B * C * L.nbands);
    L.work = take(sizeof(int) * (size_t)B * C * L.nbands);
    L.work_ctr = take(sizeof(int) * 4);
    L.cand_key = take(sizeof(int) * (size_t)B * L.cand_cap);
    L.cand_val = take(sizeof(int) * (size_t)B * L.cand_cap);
    L.cand_n = take(sizeof(int) * (size_t)B);
    L.cand_data = take(sizeof(float4) * (size_t)B * L.cand_cap);
    L.votes = want_votes ? take(sizeof(float) * (size_t)B * C * HW) : o;
    L.total = o;
    return L;
}

// ----------------------------------------------------------------------------------------
// geometry shared by the kernels (formulas of .cu.cc:32-42, 73-172 with the rounding that
// nvcc's default contraction gives the reference: a*b + c*d -> fma(a, b, RN(c*d)))
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ float project_box(int cls, const float* __restrict__ extents,
                                             const float* __restrict__ meta, float distance, float factor)
{
    float xHalf = extents[cls * 3 + 0] * 0.5f;
    float yHalf = extents[cls * 3 + 1] * 0.5f;
    float zHalf = extents[cls * 3 + 2] * 0.5f;
    float fx = meta[0], fy = meta[4], px = meta[2], py = meta[5];
    float minX = 1e8f, maxX = -1e8f, minY = 1e8f, maxY = -1e8f;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        float X = (i & 1) ? -xHalf : xHalf;
        float Y = (i & 2) ? -yHalf : yHalf;
        float Z = __fadd_rn((i & 4) ? -zHalf : zHalf, distance);
        float x = __fmaf_rn(fx, __fdiv_rn(X, Z), px);
        float y = __fmaf_rn(fy, __fdiv_rn(Y, Z), py);
        minX = fminf(minX, x); minY = fminf(minY, y);
        maxX = fmaxf(maxX, x); maxY = fmaxf(maxY, y);
    }
    float width = __fadd_rn(__fsub_rn(maxX, minX), 1.f);
    float height = __fadd_rn(__fsub_rn(maxY, minY), 1.f);
    return __fmul_rn(fmaxf(width, height), factor);
}

// the reference predicate, bit for bit: dot / (n1 * n2) > inlier  (angle_distance, .cu.cc:32-42)
__device__ __forceinline__ bool pred_exact(float u, float v, float n1, float dx, float dy, float inlier)
{
    float n2 = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    float dot = __fmaf_rn(u, dx, __fmul_rn(v, dy));
    float c = __fdiv_rn(dot, __fmul_rn(n1, n2));
    return c > inlier;
}

// same decision, cheap: sign of dot - inlier*n1*|d| when it is far (4e-6 relative) from zero,
// otherwise the exact evaluation.  vdy = RN(v*dy), dy2 = dy*dy, tn1 = inlier*n1.
__device__ __forceinline__ bool pred_fast(float u, float v, float n1, float tn1, float dx, float dy, float vdy,
                                          float dy2, float inlier)
{
    float s2 = __fmaf_rn(dx, dx, dy2);
    float dot = __fmaf_rn(u, dx, vdy);
    float rhs = tn1 * (s2 * rsqrtf(s2));
    float g = dot - rhs;
    if (fabsf(g) > 4e-6f * rhs) return g > 0.f;
    return pred_exact(u, v, n1, dx, dy, inlier);
}

// ----------------------------------------------------------------------------------------
// k_hist: per-chunk class histogram; also zero-fills the five output buffers + counters
// ----------------------------------------------------------------------------------------
struct ZeroList {
    float* p[5];
    unsigned n[5];
};

__global__ void __launch_bounds__(kThreads)
k_hist(const int* __restrict__ label, int HW, int C, int nchunks, int* __restrict__ chunk_hist, int* __restrict__ cls_size,
       int* __restrict__ bbox, int* __restrict__ cand_n, int* __restrict__ work_ctr, ZeroList z)
{
    extern __shared__ int sh[];
    const int b = blockIdx.y, chunk = blockIdx.x, t = threadIdx.x, lane = t & 31;
    // zero-fill outputs (reset_outputs, .cu.cc:579-588), spread over the whole grid
    {
        unsigned gid = (blockIdx.y * gridDim.x + blockIdx.x) * kThreads + t;
        unsigned gsz = gridDim.x * gridDim.y * kThreads;
#pragma unroll
        for (int k = 0; k < 5; k++)
            for (unsigned i = gid; i < z.n[k]; i += gsz) z.p[k][i] = 0.f;
    }
    if (chunk == 0) {  // per-image state consumed by the later kernels
        for (int c = t; c < C; c += kThreads) {
            int* bb = bbox + ((size_t)b * C + c) * 4;
            bb[0] = 0x7fffffff; bb[1] = -1; bb[2] = 0x7fffffff; bb[3] = -1;
        }
        if (t == 0) {
            cand_n[b] = 0;
            if (b == 0) { work_ctr[0] = 0; work_ctr[1] = 0; }
        }
    }
    for (int c = t; c < C; c += kThreads) sh[c] = 0;
    __syncthreads();
    const int* lab = label + (size_t)b * HW;
#pragma unroll
    for (int j = 0; j < kChunk / kThreads; j++) {
        int p = chunk * kChunk + j * kThreads + t;
        int cls = p < HW ? lab[p] : -1;
        bool valid = cls > 0 && cls < C;
        unsigned peers = __match_any_sync(0xffffffffu, valid ? cls : -1);
        if (valid && lane == __ffs(peers) - 1) atomicAdd(&sh[cls], __popc(peers));
    }
    __syncthreads();
    int* out = chunk_hist + ((size_t)b * nchunks + chunk) * C;
    for (int c = t; c < C; c += kThreads) {
        int v = sh[c];
        out[c] = v;
        if (v) atomicAdd(&cls_size[b * C + c], v);  // class totals (zeroed by the host-side memset node)
    }
}

// ----------------------------------------------------------------------------------------
// k_emit: canonical (ascending pixel index) rank of every foreground pixel within its class;
// pixels with rank % skip == 0 become samples (the sub-sampling of .cu.cc:269 applied to the
// canonical list order of SURVEY.md §8(c))
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_emit(const int* __restrict__ label, const VertexSrc vsrc, const float* __restrict__ extents,
       const float* __restrict__ meta_all, int H, int W, int C, int num_meta, int nchunks, int skip, int label_thr,
       float inlier, const int* __restrict__ chunk_hist, const int* __restrict__ cls_size, int* __restrict__ cls_slot,
       int* __restrict__ cls_nsamp, int* __restrict__ cls_soff, int* __restrict__ slot_cls, int* __restrict__ img_count,
       Sample* __restrict__ samples, int samp_cap, int* __restrict__ bbox)
{
    // smem: [kWarps][C] warp histograms | [C][4] block bounding boxes | [C] slot | [C] sample offset | [C] chunk prefix
    //       | [kChunk] int2 sample queue
    extern __shared__ int wh[];
    const int b = blockIdx.y, chunk = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int HW = H * W;
    int* sbb = wh + kWarps * C;
    int* s_slot = sbb + 4 * C;
    int* s_soff = s_slot + C;
    int* s_pref = s_soff + C;
    // class table of this image (class_indexes of .cu.cc:650-663): classes with more than label_thr pixels,
    // ascending; sample offsets = running sum of ceil(size / skip).  Every CTA recomputes it (C is small),
    // the CTA of chunk 0 publishes it for the later kernels.
    if (w == 0) {
        int slot_run = 0, soff_run = 0;
        for (int c0 = 0; c0 < C; c0 += 32) {
            const int c = c0 + lane;
            const int sz = c < C ? cls_size[b * C + c] : 0;
            const bool present = c > 0 && c < C && sz > label_thr;
            const int ns = present ? (sz + skip - 1) / skip : 0;
            const unsigned pm = __ballot_sync(0xffffffffu, present);
            int incl = ns;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int nb = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += nb;
            }
            const int slot = slot_run + __popc(pm & ((1u << lane) - 1u));
            const int soff = soff_run + incl - ns;
            if (c < C) {
                s_slot[c] = present ? slot : -1;
                s_soff[c] = soff;
                if (chunk == 0) {
                    cls_slot[b * C + c] = present ? slot : -1;
                    cls_nsamp[b * C + c] = ns;
                    cls_soff[b * C + c] = present ? soff : 0;
                    if (present) slot_cls[b * C + slot] = c;
                }
            }
            slot_run += __popc(pm);
            soff_run += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (chunk == 0 && lane == 0) img_count[b] = slot_run;
    }
    for (int i = t; i < kWarps * C; i += kThreads) wh[i] = 0;
    for (int i = t; i < C; i += kThreads) { sbb[4 * i] = 0x7fffffff; sbb[4 * i + 1] = -1; sbb[4 * i + 2] = 0x7fffffff; sbb[4 * i + 3] = -1; }
    __syncthreads();
    // pixels of this class in earlier chunks of the image (one warp per class, lanes over chunks)
    for (int c = w; c < C; c += kWarps) {
        int sum = 0;
        if (s_slot[c] >= 0)
            for (int k = lane; k < chunk; k += 32) sum += chunk_hist[((size_t)b * nchunks + k) * C + c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) s_pref[c] = sum;
    }
    const int* lab = label + (size_t)b * HW;
    const int base = chunk * kChunk + w * (kChunk / kWarps);
    int labs[kChunk / kThreads];
#pragma unroll
    for (int s = 0; s < kChunk / kThreads; s++) {
        int p = base + s * 32 + lane;
        int cls = p < HW ? lab[p] : -1;
        if (!(cls > 0 && cls < C) || s_slot[cls] < 0) cls = -1;
        labs[s] = cls;
    }
#pragma unroll
    for (int s = 0; s < kChunk / kThreads; s++) {
        int cls = labs[s];
        unsigned peers = __match_any_sync(0xffffffffu, cls);
        if (cls >= 0 && lane == __ffs(peers) - 1) wh[w * C + cls] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    for (int c = t; c < C; c += kThreads) {
        int run = s_pref[c];
#pragma unroll
        for (int ww = 0; ww < kWarps; ww++) {
            int tmp = wh[ww * C + c];
            wh[ww * C + c] = run;
            run += tmp;
        }
    }
    __syncthreads();
    const float* meta = meta_all + (size_t)b * num_meta;
    const unsigned lt = (1u << lane) - 1u;
    // pass 2: ranks; sampled pixels are queued in shared memory so that the (divergent, ~600
    // instruction) record construction below runs on densely packed lanes
    int2* queue = reinterpret_cast<int2*>(wh + (((kWarps + 7) * C + 1) & ~1));  // [kChunk] (pixel offset in chunk | class << 16, sample index)
    __shared__ int s_qn;
    if (t == 0) s_qn = 0;
    __syncthreads();
#pragma unroll
    for (int s = 0; s < kChunk / kThreads; s++) {
        int cls = labs[s];
        unsigned peers = __match_any_sync(0xffffffffu, cls);
        int rank = 0;
        if (cls >= 0) rank = wh[w * C + cls] + __popc(peers & lt);
        __syncwarp();
        if (cls >= 0 && lane == __ffs(peers) - 1) wh[w * C + cls] += __popc(peers);
        __syncwarp();
        if (cls >= 0 && rank % skip == 0) {
            int pos = atomicAdd(&s_qn, 1);
            queue[pos] = make_int2((w * (kChunk / kWarps) + s * 32 + lane) | (cls << 16), rank / skip);
        }
    }
    __syncthreads();
    const int qn = s_qn;
    for (int qi = t; qi < qn; qi += kThreads) {
        const int2 qe = queue[qi];
        const int cls = qe.x >> 16;
        const int p = chunk * kChunk + (qe.x & 0xffff);
        {
            int x = p % W, y = p / W;
            float u, v, z;
            if (vsrc.dense) {
                size_t off = (size_t)3 * cls + (size_t)3 * C * ((size_t)b * HW + p);
                u = vsrc.dense[off]; v = vsrc.dense[off + 1]; z = vsrc.dense[off + 2];
            } else {
                const int ch = C + 3 * cls;   // lowres channel of vertex_pred channel 3 cls
                u = up8_value(vsrc.lowres, b, vsrc.h, vsrc.w, 4 * C, ch, y, x, __ldg(vsrc.bias + 3 * cls));
                v = up8_value(vsrc.lowres, b, vsrc.h, vsrc.w, 4 * C, ch + 1, y, x, __ldg(vsrc.bias + 3 * cls + 1));
                z = up8_value(vsrc.lowres, b, vsrc.h, vsrc.w, 4 * C, ch + 2, y, x, __ldg(vsrc.bias + 3 * cls + 2));
            }
            float d = expf(z);
            const float s2 = __fmaf_rn(u, u, __fmul_rn(v, v));
            float n1 = __fsqrt_rn(s2);
            float thr = project_box(cls, extents, meta, d, 0.6f);
            // (u, v) != 0 but u*u + v*v underflows to n1 = 0: the reference's dot / (n1 * n2) is +-inf, so the pixel
            // votes for every cell of its window with dot > 0, a half-plane
            const bool half = n1 == 0.f && (u != 0.f || v != 0.f);
            int m = -1;
            if (thr == thr && (n1 > 0.f || half) && n1 < INFINITY) {
                float mf = fminf(fmaxf(ceilf(thr) - 1.f, -1.f), (float)kMaxM);
                m = (int)mf;
            }
            // boundary rays of the cone: axis rotated by +-acos(inlier)
            float inv = 1.f / n1, uh = u * inv, vh = v * inv;
            float ca = inlier;
            // u*u + v*v subnormal: n1 = sqrt(s2) carries the rounding of a subnormal (up to ~50% near the bottom of the
            // range, ~1% at |(u, v)| = 1e-22), so the reference's cone is cos > inlier * n1 / |(u, v)|.  The rays are
            // built from that threshold and the direction normalised in scaled arithmetic (2^64: exact, and |(u, v)| >=
            // 2^-75 here), and flag 256 has k_vote re-check every end point of the sample with the reference predicate.
            const bool sub = s2 > 0.f && s2 < FLT_MIN;
            if (sub) {
                const float us = u * 0x1p64f, vs = v * 0x1p64f, ns = sqrtf(us * us + vs * vs);
                uh = us / ns;
                vh = vs / ns;
                ca = fminf(inlier * (n1 * 0x1p64f) / ns, 1.f);
            }
            float sa = sqrtf(fmaxf(1.f - ca * ca, 0.f));
            float r1x = ca * uh - sa * vh, r1y = ca * vh + sa * uh;
            float r2x = ca * uh + sa * vh, r2y = ca * vh - sa * uh;
            float k1 = r1x / r1y, k2 = r2x / r2y;
            int flags = (r1y > 0.f ? 1 : 0) | (r1y < 0.f ? 2 : 0) | (r2y > 0.f ? 4 : 0) | (r2y < 0.f ? 8 : 0) |
                        ((r2x - r2y * k1) > 0.f ? 16 : 0) | ((r1x - r1y * k2) > 0.f ? 32 : 0) |
                        (pred_exact(u, v, n1, 1.f, 0.f, inlier) ? 64 : 0) | (pred_exact(u, v, n1, -1.f, 0.f, inlier) ? 128 : 0) |
                        (sub ? 256 : 0);
            if (half) {
                // one boundary line dot = 0, dx = dy * (-v / u), for rows above and below; the voted cells lie on the
                // side u points to.  u == 0: dot = v * dy, whole rows on the side v points to (k1 = -inf there puts
                // the line's crossing at -infinity, so the single-ray case below opens the interval over the row).
                // The own-row flags are already the reference's (dot = u * dx).
                k1 = k2 = u != 0.f ? -v / u : (v > 0.f ? -INFINITY : INFINITY);
                flags = (flags & (64 | 128)) | (u != 0.f ? 1 | 2 : (v > 0.f ? 1 : 2)) | (u >= 0.f ? 16 : 0);
            }
            Sample rec;
            rec.xy = x | (y << 16);
            rec.u = u; rec.v = v; rec.n1 = n1; rec.k1 = k1; rec.k2 = k2;
            rec.mflags = (m & 0xffff) | (flags << 16);
            rec.d = d;
            Sample* dst = samples + (size_t)b * samp_cap + s_soff[cls] + qe.y;
            reinterpret_cast<float4*>(dst)[0] = reinterpret_cast<const float4*>(&rec)[0];
            reinterpret_cast<float4*>(dst)[1] = reinterpret_cast<const float4*>(&rec)[1];
            if (m >= 0) {
                atomicMin(&sbb[4 * cls + 0], max(y - m, 0));
                atomicMax(&sbb[4 * cls + 1], min(y + m, H - 1));
                atomicMin(&sbb[4 * cls + 2], max(x - m, 0));
                atomicMax(&sbb[4 * cls + 3], min(x + m, W - 1));
            }
        }
    }
    __syncthreads();
    for (int c = t; c < C; c += kThreads)
        if (sbb[4 * c + 1] >= 0) {
            int* bb = bbox + ((size_t)b * C + c) * 4;
            atomicMin(&bb[0], sbb[4 * c]);
            atomicMax(&bb[1], sbb[4 * c + 1]);
            atomicMin(&bb[2], sbb[4 * c + 2]);
            atomicMax(&bb[3], sbb[4 * c + 3]);
        }
}

// ----------------------------------------------------------------------------------------
// k_worklist: (image, slot, band) items for every band that intersects a class's vote box
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
k_worklist(int B, int C, int R, int nbands, const int* __restrict__ img_count, const int* __restrict__ slot_cls,
           const int* __restrict__ cls_nsamp, const int* __restrict__ bbox, int* __restrict__ work,
           int* __restrict__ work_ctr)
{
    // Items are laid out by (coarsely) descending sample count of their class: longest first keeps the
    // persistent k_vote CTAs balanced.  The order has no effect on results.  Counting sort on 64 buckets.
    __shared__ int s_cnt[64];
    __shared__ int s_base[64];
    const int n = B * C;
    if (threadIdx.x < 64) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    auto bucket = [](int ns) { return 63 - min(63, ns >> 8); };  // 256 samples per bucket, big classes first
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int b = i / C, slot = i % C;
        if (slot >= img_count[b]) continue;
        int c = slot_cls[b * C + slot];
        const int* bb = bbox + ((size_t)b * C + c) * 4;
        if (bb[1] < bb[0]) continue;
        atomicAdd(&s_cnt[bucket(cls_nsamp[b * C + c])], bb[1] / R - bb[0] / R + 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int k = 0; k < 64; k++) { s_base[k] = run; run += s_cnt[k]; }
        work_ctr[0] = 0; work_ctr[1] = run;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int b = i / C, slot = i % C;
        if (slot >= img_count[b]) continue;
        int c = slot_cls[b * C + slot];
        const int* bb = bbox + ((size_t)b * C + c) * 4;
        if (bb[1] < bb[0]) continue;
        int lo = bb[0] / R, nb = bb[1] / R - lo + 1;
        int pos = atomicAdd(&s_base[bucket(cls_nsamp[b * C + c])], nb);
        for (int k = 0; k < nb; k++) work[pos + k] = (b * C + slot) * nbands + lo + k;
    }
}

// ----------------------------------------------------------------------------------------
// k_vote: persistent CTAs; one (image, class, band) difference array in shared memory
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 4)
k_vote(int H, int W, int C, int R, int nbands, float inlier, float tau0, const int* __restrict__ slot_cls,
       const int* __restrict__ cls_nsamp, const int* __restrict__ cls_soff, const int* __restrict__ bbox,
       const Sample* __restrict__ samples, int samp_cap, const int* __restrict__ work, int* __restrict__ work_ctr,
       int2* __restrict__ band_res, float* __restrict__ votes_out)
{
    extern __shared__ int D[];
    __shared__ int s_item;
    __shared__ int s_red_val[kWarps];
    __shared__ int s_red_idx[kWarps];
    __shared__ int4 s_q[kWarps][64];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int total = work_ctr[1];
    // R (rows per band) is a power of two <= 32
    while (true) {
        __syncthreads();
        if (t == 0) s_item = atomicAdd(&work_ctr[0], 1);
        __syncthreads();
        const int item = s_item;
        if (item >= total) break;
        const int key = work[item];
        const int band = key % nbands, bs = key / nbands, slot = bs % C, b = bs / C;
        const int c = slot_cls[b * C + slot];
        const int* bb = bbox + ((size_t)b * C + c) * 4;
        const int xlo = bb[2], xhi = bb[3];
        const int Wd = xhi - xlo + 1;
        const int stride = (Wd + 1) | 1;
        const int r0 = band * R;
        const int nrows = min(R, H - r0);
        for (int i = t; i < R * stride; i += kThreads) D[i] = 0;
        __syncthreads();

        const int ns = cls_nsamp[b * C + c];
        const Sample* S = samples + (size_t)b * samp_cap + cls_soff[b * C + c];
        int4* Q = s_q[w];   // this warp's queue of (sample, row) pairs whose end points need the exact check
        int qn = 0;         // warp-uniform
        const unsigned lt = (1u << lane) - 1u;

        // Re-check of queued pairs with the reference predicate, on densely packed lanes.
        auto drain = [&](int count) {
            if (lane < count) {
                const int4 q = Q[lane];
                const Sample* rp = S + q.x;
                const float4 q0 = __ldg(reinterpret_cast<const float4*>(rp));
                const int mfl = __float_as_int(__ldg(reinterpret_cast<const float*>(rp) + 6));
                const int xy = __float_as_int(q0.x);
                const int x = xy & 0xffff, y = xy >> 16, m = (int)(short)(mfl & 0xffff);
                const int row = q.y & 0xff, mode = q.y >> 8;
                const float u = q0.y, v = q0.z, n1 = q0.w;
                const float dy = (float)(r0 + row - y);
                const int wmin = max(x - m, 0), wmax = min(x + m, W - 1);
                const float tn1 = inlier * n1, vdy = __fmul_rn(v, dy), dy2 = dy * dy;
                auto P = [&](int cx) { return pred_fast(u, v, n1, tn1, (float)(cx - x), dy, vdy, dy2, inlier); };
                int a = q.z, e = q.w;
                bool ok = true;
                if (mode & 12) {
                    ok = false;
                    if ((mode & 4) && P(a)) { e = a; ok = true; }
                    else if ((mode & 8) && P(e)) { a = e; ok = true; }
                } else {
#pragma unroll 1
                    for (int side = 0; side < 2 && ok; side++) {
                        if (!(mode & (1 << side))) continue;
                        const int o = side ? 1 : -1, lim = side ? wmax : wmin;
                        int pc = side ? e : a;
                        while (pc != lim && P(pc + o)) pc += o;                        // grow outwards while cells pass
                        while ((side ? pc >= a : pc <= e) && !P(pc)) pc -= o;          // shrink inwards while they fail
                        if (side) e = pc; else a = pc;
                        ok = a <= e;
                    }
                }
                if (ok) {
                    int* Dq = D + row * stride - xlo;
                    atomicAdd(&Dq[a], 1);
                    atomicAdd(&Dq[e + 1], -1);
                }
            }
            __syncwarp();
        };

        // lane = sample: 32 samples per warp iteration, each lane walks the R rows of the band with a per-lane
        // rotation of the start row, so that at any moment the lanes touch different rows of the difference array.
        // The record decode, the reach test and the bounds are done once per (sample, band) instead of once per
        // (sample, row); warps whose 32 samples (consecutive in raster order) do not reach the band leave at once.
        // The record of the next iteration is in flight while this one is processed.
        int sidx = w * 32 + lane;
        float4 n0 = make_float4(0, 0, 0, 0), n1v = n0;
        if (sidx < ns) {
            n0 = __ldg(reinterpret_cast<const float4*>(S + sidx));
            n1v = __ldg(reinterpret_cast<const float4*>(S + sidx) + 1);
        }
        for (int sb = w * 32; sb < ns; sb += kWarps * 32) {
            const float4 q0 = n0, q1 = n1v;
            const int scur = sidx;
            sidx += kWarps * 32;
            if (sidx < ns) {
                n0 = __ldg(reinterpret_cast<const float4*>(S + sidx));
                n1v = __ldg(reinterpret_cast<const float4*>(S + sidx) + 1);
            }
            const int xy = __float_as_int(q0.x);
            const int x = xy & 0xffff, y = xy >> 16;
            const int mflags = __float_as_int(q1.z);
            const int m = (int)(short)(mflags & 0xffff);
            const int fl = mflags >> 16;
            // rows of the band this sample reaches: |cy - y| <= m
            const int row_lo = max(y - m, r0) - r0, row_hi = min(y + m, r0 + nrows - 1) - r0;
            const bool reach = scur < ns && m >= 0 && row_lo <= row_hi;
            if (!__any_sync(0xffffffffu, reach)) continue;
            const int wmin = max(x - m, 0), wmax = min(x + m, W - 1);
            // flag 256: every end point of this sample is re-checked (the m^2 term then puts tau far above 1)
            const float fm2 = (fl & 256) ? 1e12f : (float)(m * m);
#pragma unroll 1
            for (int k = 0; k < R; k++) {
                const int rl = (lane + k) & (R - 1);
                const int idy = r0 + rl - y;
                int act = 0;      // 0 nothing, 1 interval [a, e] trusted, 2 queued for the exact check
                int a = 0, e = 0, mode = 0;
                if (reach && rl >= row_lo && rl <= row_hi) {
                    if (idy == 0) {
                        // the pixel's own row: cos = sign(dx) * u / n1, decided once per sample in k_emit
                        if (fl & 64) { a = x + 1; e = wmax; act = a <= e; }
                        else if (fl & 128) { a = wmin; e = x - 1; act = a <= e; }
                    } else {
                        const bool v1 = idy > 0 ? (fl & 1) : (fl & 2);
                        const bool v2 = idy > 0 ? (fl & 4) : (fl & 8);
                        if (v1 || v2) {
                            const float dy = (float)idy;
                            const float h1 = dy * q1.x, h2 = dy * q1.y;
                            float lo, hi;
                            if (v1 && v2) { lo = fminf(h1, h2); hi = fmaxf(h1, h2); }
                            else {
                                const float hh = v1 ? h1 : h2;
                                const bool up = v1 ? (fl & 16) : (fl & 32);
                                lo = up ? hh : -1e9f;
                                hi = up ? 1e9f : hh;
                            }
                            lo = fminf(fmaxf(lo, -40000.f), 40000.f);
                            hi = fminf(fmaxf(hi, -40000.f), 40000.f);
                            a = x + (int)ceilf(lo);
                            e = x + (int)floorf(hi);
                            // The ray estimate and the fp32 predicate both sit within ~1e-6 (dy^2 + m^2) / |dy| cells
                            // of the real cone boundary (DESIGN.md §3.3); an end point closer than tau to an integer
                            // is re-checked with the reference predicate, the others are exact as they are.
                            const float tau = tau0 + 2e-6f * __fdividef(dy * dy + fm2, fabsf(dy));
                            if (a > e) {
                                const bool ca = (float)(a - x) - hi < tau && a >= wmin && a <= wmax;
                                const bool ce = lo - (float)(e - x) < tau && e >= wmin && e <= wmax;
                                if (ca || ce) { act = 2; mode = (ca ? 4 : 0) | (ce ? 8 : 0); }
                            } else {
                                const float ma = (float)(a - x) - lo, me = hi - (float)(e - x);
                                const bool va = a >= wmin && (ma < tau || ma > 1.f - tau);
                                const bool ve = e <= wmax && (me < tau || me > 1.f - tau);
                                const int chk = (va || ve) ? 1 : 0;
                                a = max(a, wmin);
                                e = min(e, wmax);
                                // a == e + 1 with a checked end point: the estimate starts (ends) within rounding distance of
                                // the window edge, just outside it; the exact check grows it back over the edge cell
                                if (a <= e + chk) { act = 1 + chk; mode = (va ? 1 : 0) | (ve ? 2 : 0); }
                            }
                        }
                    }
                }
                if (act == 1) {
                    int* Drow = D + rl * stride - xlo;
                    atomicAdd(&Drow[a], 1);
                    atomicAdd(&Drow[e + 1], -1);
                }
                const unsigned need = __ballot_sync(0xffffffffu, act == 2);
                if (need) {
                    if (act == 2) Q[qn + __popc(need & lt)] = make_int4(scur, rl | (mode << 8), a, e);
                    qn += __popc(need);
                    __syncwarp();
                    if (qn >= 32) {
                        drain(32);
                        if (lane < qn - 32) Q[lane] = Q[32 + lane];
                        qn -= 32;
                        __syncwarp();
                    }
                }
            }
        }
        if (qn > 0) drain(qn);
        __syncthreads();

        // row prefix sums fused with the arg-max (first maximum in flat index order)
        int best_val = -1, best_idx = 0x7fffffff;
        for (int row = w; row < nrows; row += kWarps) {
            int carry = 0;
            int* Dr = D + row * stride;
            for (int x0 = 0; x0 < Wd; x0 += 32) {
                int xi = x0 + lane;
                int val = xi < Wd ? Dr[xi] : 0;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    int nb = __shfl_up_sync(0xffffffffu, val, o);
                    if (lane >= o) val += nb;
                }
                val += carry;
                carry = __shfl_sync(0xffffffffu, val, 31);
                if (xi < Wd) {
                    if (votes_out) Dr[xi] = val;
                    int idx = (r0 + row) * W + xlo + xi;
                    if (val > best_val) { best_val = val; best_idx = idx; }
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            int ov = __shfl_xor_sync(0xffffffffu, best_val, o);
            int oi = __shfl_xor_sync(0xffffffffu, best_idx, o);
            if (ov > best_val || (ov == best_val && oi < best_idx)) { best_val = ov; best_idx = oi; }
        }
        if (lane == 0) { s_red_val[w] = best_val; s_red_idx[w] = best_idx; }
        __syncthreads();
        if (t == 0) {
            int bv = s_red_val[0], bi = s_red_idx[0];
            for (int k = 1; k < kWarps; k++)
                if (s_red_val[k] > bv || (s_red_val[k] == bv && s_red_idx[k] < bi)) { bv = s_red_val[k]; bi = s_red_idx[k]; }
            band_res[(size_t)(b * C + slot) * nbands + band] = make_int2(bv, bi);
        }
        if (votes_out) {
            float* plane = votes_out + ((size_t)b * C + c) * H * W;
            for (int i = t; i < nrows * W; i += kThreads) {
                int row = i / W, x = i % W;
                float val = (x >= xlo && x <= xhi) ? (float)D[row * stride + x - xlo] : 0.f;
                plane[(size_t)(r0 + row) * W + x] = val;
            }
        }
    }
}

// ----------------------------------------------------------------------------------------
// k_select: default mode — first arg-max of each present class (thrust::max_element,
// .cu.cc:752-762), first `cap` classes (.cu.cc:773-774)
// ----------------------------------------------------------------------------------------
__global__ void k_select(int C, int HW, int R, int nbands, int cap, int cand_cap, const int* __restrict__ img_count,
                         const int* __restrict__ slot_cls, const int* __restrict__ bbox,
                         const int2* __restrict__ band_res, int* __restrict__ cand_key, int* __restrict__ cand_val,
                         int* __restrict__ cand_n)
{
    const int b = blockIdx.x;
    const int count = img_count[b];
    const int n = min(min(count, cap), cand_cap);
    for (int slot = threadIdx.x; slot < n; slot += blockDim.x) {
        int c = slot_cls[b * C + slot];
        const int* bb = bbox + ((size_t)b * C + c) * 4;
        int bv = 0, bi = 0;
        if (bb[1] >= bb[0]) {
            int lo = bb[0] / R, hi = bb[1] / R;
            bv = -1; bi = 0x7fffffff;
            for (int k = lo; k <= hi; k++) {
                int2 r = band_res[(size_t)(b * C + slot) * nbands + k];
                if (r.x > bv || (r.x == bv && r.y < bi)) { bv = r.x; bi = r.y; }
            }
            if (bv <= 0) { bv = 0; bi = 0; }  // empty plane: max_element returns the first element
        }
        cand_key[(size_t)b * cand_cap + slot] = slot * HW + bi;
        cand_val[(size_t)b * cand_cap + slot] = bv;
    }
    if (threadIdx.x == 0) cand_n[b] = n;
}

// ----------------------------------------------------------------------------------------
// k_localmax: threshold mode — vote > threshold and no strictly greater vote in the clipped
// 7x7 window (.cu.cc:351-367); the box / density tests need hough_data and run in k_finalize
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_localmax(int H, int W, int C, int R, float vote_thr, int cand_cap, const int* __restrict__ img_count,
           const int* __restrict__ slot_cls, const int* __restrict__ bbox, const float* __restrict__ votes,
           int* __restrict__ cand_key, int* __restrict__ cand_val, int* __restrict__ cand_n, int* __restrict__ status)
{
    const int b = blockIdx.z, slot = blockIdx.y;
    if (slot >= img_count[b]) return;
    const int c = slot_cls[b * C + slot];
    const int* bb = bbox + ((size_t)b * C + c) * 4;
    if (bb[1] < bb[0]) return;
    const int ylo = (bb[0] / R) * R, yhi = min(H - 1, (bb[1] / R) * R + R - 1);  // rows written by k_vote
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= H * W) return;
    const int cx = p % W, cy = p / W;
    if (cy < ylo || cy > yhi) return;
    const float* plane = votes + ((size_t)b * C + c) * H * W;
    const float val = plane[p];
    if (!(val > vote_thr)) return;
    for (int x = cx - 3; x <= cx + 3; x++)
        for (int y = cy - 3; y <= cy + 3; y++)
            if (x >= 0 && x < W && y >= ylo && y <= yhi && plane[y * W + x] > val) return;
    int pos = atomicAdd(&cand_n[b], 1);
    if (pos < cand_cap) {
        cand_key[(size_t)b * cand_cap + pos] = slot * (H * W) + p;
        cand_val[(size_t)b * cand_cap + pos] = (int)val;
    } else if (status) {
        atomicOr(&status[0], 1);
    }
}

// ----------------------------------------------------------------------------------------
// k_celldata: per candidate cell, the reference's per-cell loops (.cu.cc:266-331): exact
// recount, mean depth, second pass for the box extents
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_celldata(int B, int H, int W, int C, int num_meta, float inlier, int cand_cap, const float* __restrict__ extents,
           const float* __restrict__ meta_all, const int* __restrict__ slot_cls, const int* __restrict__ cls_nsamp,
           const int* __restrict__ cls_soff, const Sample* __restrict__ samples, int samp_cap,
           const int* __restrict__ cand_key, const int* __restrict__ cand_n, float4* __restrict__ cand_data)
{
    __shared__ float s_sum[kThreads];
    __shared__ int s_cnt[kThreads];
    __shared__ float s_thr2;
    const int t = threadIdx.x;
    const int HW = H * W;
    {
        const int b = blockIdx.y;  // grid = (candidate lanes per image, B)
        const int n = min(cand_n[b], cand_cap);
        for (int i = blockIdx.x; i < n; i += gridDim.x) {
            const int key = cand_key[(size_t)b * cand_cap + i];
            const int slot = key / HW, p = key % HW;
            const int c = slot_cls[b * C + slot];
            const int cx = p % W, cy = p / W;
            const int ns = cls_nsamp[b * C + c];
            const Sample* S = samples + (size_t)b * samp_cap + cls_soff[b * C + c];
            float sum = 0.f;
            int cnt = 0;
            for (int s = t; s < ns; s += kThreads) {
                const Sample q = S[s];
                const int x = q.xy & 0xffff, y = q.xy >> 16;
                const int m = (int)(short)(q.mflags & 0xffff);
                if (m < 0 || abs(x - cx) > m || abs(y - cy) > m) continue;
                if (pred_exact(q.u, q.v, q.n1, (float)(cx - x), (float)(cy - y), inlier)) { cnt++; sum += q.d; }
            }
            s_sum[t] = sum; s_cnt[t] = cnt;
            __syncthreads();
            for (int o = kThreads / 2; o > 0; o >>= 1) {
                if (t < o) { s_sum[t] += s_sum[t + o]; s_cnt[t] += s_cnt[t + o]; }
                __syncthreads();
            }
            const int votes = s_cnt[0];
            float dist = 0.f;
            if (votes > 0) dist = __fdiv_rn(s_sum[0], (float)votes);
            if (t == 0) s_thr2 = votes > 0 ? project_box(c, extents, meta_all + (size_t)b * num_meta, dist, 0.6f) : 0.f;
            __syncthreads();
            const float thr2 = s_thr2;
            float bbw = -1.f, bbh = -1.f;
            if (votes > 0) {
                for (int s = t; s < ns; s += kThreads) {
                    const Sample q = S[s];
                    const int x = q.xy & 0xffff, y = q.xy >> 16;
                    const float dx = fabsf((float)(x - cx)), dy = fabsf((float)(y - cy));
                    if (!(dx < thr2 && dy < thr2)) continue;
                    if (pred_exact(q.u, q.v, q.n1, (float)(cx - x), (float)(cy - y), inlier)) {
                        bbw = fmaxf(bbw, dx);
                        bbh = fmaxf(bbh, dy);
                    }
                }
            }
            __syncthreads();
            s_sum[t] = bbw;
            reinterpret_cast<float*>(s_cnt)[t] = bbh;
            __syncthreads();
            for (int o = kThreads / 2; o > 0; o >>= 1) {
                if (t < o) {
                    s_sum[t] = fmaxf(s_sum[t], s_sum[t + o]);
                    reinterpret_cast<float*>(s_cnt)[t] =
                        fmaxf(reinterpret_cast<float*>(s_cnt)[t], reinterpret_cast<float*>(s_cnt)[t + o]);
                }
                __syncthreads();
            }
            if (t == 0) {
                float4 r;
                if (votes > 0) {
                    r.x = dist;
                    r.y = 2.f * reinterpret_cast<float*>(s_cnt)[0];
                    r.z = 2.f * s_sum[0];
                } else {
                    r.x = 0.f; r.y = 0.f; r.z = 0.f;  // hough_data stays zero (.cu.cc:296)
                }
                r.w = (float)votes;
                cand_data[(size_t)b * cand_cap + i] = r;
            }
            __syncthreads();
        }
    }
}

// ----------------------------------------------------------------------------------------
// k_finalize: ROI cap, row offsets, rows (compute_rois_kernel, .cu.cc:386-576)
// ----------------------------------------------------------------------------------------
__device__ float box_overlap(int cls, const float* __restrict__ extents, const float* __restrict__ meta,
                             const float* __restrict__ pose, const float* box)
{
    // compute_box_overlap, .cu.cc:123-172: rotate the 8 extent corners by the gt quaternion
    // (unit-quaternion rotation matrix), translate, project, IoU with the predicted box
    float xHalf = extents[cls * 3 + 0] * 0.5f, yHalf = extents[cls * 3 + 1] * 0.5f, zHalf = extents[cls * 3 + 2] * 0.5f;
    float w = pose[6], x = pose[7], y = pose[8], z = pose[9];
    float tx = 2 * x, ty = 2 * y, tz = 2 * z;
    float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y,
          tzz = tz * z;
    float R0 = 1 - (tyy + tzz), R1 = txy - twz, R2 = txz + twy, R3 = txy + twz, R4 = 1 - (txx + tzz), R5 = tyz - twx,
          R6 = txz - twy, R7 = tyz + twx, R8 = 1 - (txx + tyy);
    float fx = meta[0], fy = meta[4], px = meta[2], py = meta[5];
    float x1 = 1e8f, x2 = -1e8f, y1 = 1e8f, y2 = -1e8f;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        float bx = (i & 1) ? -xHalf : xHalf, by = (i & 2) ? -yHalf : yHalf, bz = (i & 4) ? -zHalf : zHalf;
        float X = __fmaf_rn(R2, bz, __fmaf_rn(R1, by, R0 * bx)) + pose[10];
        float Y = __fmaf_rn(R5, bz, __fmaf_rn(R4, by, R3 * bx)) + pose[11];
        float Z = __fmaf_rn(R8, bz, __fmaf_rn(R7, by, R6 * bx)) + pose[12];
        float xx = __fmaf_rn(fx, __fdiv_rn(X, Z), px), yy = __fmaf_rn(fy, __fdiv_rn(Y, Z), py);
        x1 = fminf(x1, xx); y1 = fminf(y1, yy); x2 = fmaxf(x2, xx); y2 = fmaxf(y2, yy);
    }
    float left = fmaxf(box[0], x1), right = fminf(box[2], x2), top = fmaxf(box[1], y1), bottom = fminf(box[3], y2);
    float iw = fmaxf(right - left + 1, 0.f), ih = fmaxf(bottom - top + 1, 0.f);
    float inter = iw * ih;
    float Sa = (box[2] - box[0] + 1) * (box[3] - box[1] + 1), Sb = (x2 - x1 + 1) * (y2 - y1 + 1);
    return inter / (Sa + Sb - inter);
}

__global__ void __launch_bounds__(kThreads)
k_finalize(int B, int batch_offset, int H, int W, int C, int num_meta, int num_gt, int is_train, int cap, int cand_cap, int threshold_mode,
           float per_thr, const float* __restrict__ extents, const float* __restrict__ meta_all,
           const float* __restrict__ gt, const int* __restrict__ slot_cls, const int* __restrict__ cand_key,
           const int* __restrict__ cand_val, const int* __restrict__ cand_n, const float4* __restrict__ cand_data,
           int* __restrict__ sel /* [B][PCNN_MAX_ROI] candidate index of each kept maximum */,
           int* __restrict__ sel_n /* [B+1] counts then row offsets */, float* __restrict__ top_box,
           float* __restrict__ top_pose, float* __restrict__ top_target, float* __restrict__ top_weight,
           int* __restrict__ top_domain, int* __restrict__ num_rois, int* __restrict__ status)
{
    __shared__ int s_off[PCNN_MAX_ROI + 2];
    __shared__ int s_pass;
    const int t = threadIdx.x;
    const int HW = H * W;
    // 1. kept maxima per image, canonical order
    for (int b = 0; b < B; b++) {
        const int n = min(cand_n[b], cand_cap);
        if (!threshold_mode) {
            for (int i = t; i < n; i += kThreads) sel[b * PCNN_MAX_ROI + i] = i;
            if (t == 0) sel_n[b] = n;
        } else {
            if (t == 0) s_pass = 0;
            __syncthreads();
            for (int i = t; i < n; i += kThreads) {
                const float4 d = cand_data[(size_t)b * cand_cap + i];
                // .cu.cc:351 (box > 0) and :370 (votes / (h*w) < perThreshold rejects)
                bool pass = d.y > 0.f && d.z > 0.f && !(__fdiv_rn(d.w, d.y * d.z) < per_thr);
                if (!pass) continue;
                const int key = cand_key[(size_t)b * cand_cap + i];
                int rank = 0;
                for (int j = 0; j < n; j++) {
                    const float4 e = cand_data[(size_t)b * cand_cap + j];
                    bool pj = e.y > 0.f && e.z > 0.f && !(__fdiv_rn(e.w, e.y * e.z) < per_thr);
                    if (pj && cand_key[(size_t)b * cand_cap + j] < key) rank++;
                }
                atomicAdd(&s_pass, 1);
                if (rank < cap) sel[b * PCNN_MAX_ROI + rank] = i;
            }
            __syncthreads();
            if (t == 0) sel_n[b] = min(s_pass, cap);
            __syncthreads();
        }
    }
    __syncthreads();
    // 2. row offsets (images in order: the reference loops the batch serially, .cc:369-377)
    if (t == 0) {
        int run = 0;
        for (int b = 0; b < B; b++) { s_off[b] = run; run += sel_n[b]; }
        s_off[B] = run;
        *num_rois = run * (is_train ? 9 : 1);
    }
    __syncthreads();
    const int total = s_off[B];
    // 3. rows
    for (int r = t; r < total; r += kThreads) {
        int b = 0;
        while (s_off[b + 1] <= r) b++;
        const int i = sel[b * PCNN_MAX_ROI + (r - s_off[b])];
        const int key = cand_key[(size_t)b * cand_cap + i];
        const int slot = key / HW, p = key % HW;
        const int cls = slot_cls[b * C + slot];
        const int x = p % W, y = p / W;
        const float4 d = cand_data[(size_t)b * cand_cap + i];
        const float bb_distance = d.x, bb_height = d.y, bb_width = d.z, votes = d.w;
        if (status && (int)votes != cand_val[(size_t)b * cand_cap + i]) atomicAdd(&status[1], 1);
        const float* meta = meta_all + (size_t)b * num_meta;
        const float fx = meta[0], fy = meta[4], px = meta[2], py = meta[5];
        const float rx = __fdiv_rn((float)x - px, fx), ry = __fdiv_rn((float)y - py, fy);
        const float scale = 0.05f;
        const int nrow = is_train ? 9 : 1;
        const int roi = r * nrow;
        float* b0 = top_box + (size_t)roi * 7;
        // `x - bb_width * (0.5 + scale)` is double arithmetic in the reference (.cu.cc:417-420)
        const double f = 0.5 + (double)scale;
        b0[0] = (float)(b + batch_offset);   // global batch index (image shard of a larger batch, SURVEY.md §8(e))
        b0[1] = (float)cls;
        b0[2] = (float)((double)x - (double)bb_width * f);
        b0[3] = (float)((double)y - (double)bb_height * f);
        b0[4] = (float)((double)x + (double)bb_width * f);
        b0[5] = (float)((double)y + (double)bb_height * f);
        b0[6] = votes;
        for (int k = 0; k < nrow; k++) {
            float* q = top_pose + (size_t)(roi + k) * 7;
            q[0] = 1.f; q[1] = 0.f; q[2] = 0.f; q[3] = 0.f;
            q[4] = __fmul_rn(rx, bb_distance); q[5] = __fmul_rn(ry, bb_distance); q[6] = bb_distance;
            if (is_train) top_domain[roi + k] = num_gt == 0 ? 1 : 0;
        }
        if (!is_train) continue;
        for (int g = 0; g < num_gt; g++) {
            const float* gp = gt + (size_t)g * 13;
            if (cls == (int)gp[1] && b + batch_offset == (int)gp[0]) {
                if (box_overlap(cls, extents, meta, gp, b0 + 2) > 0.2f) {
                    for (int j = 0; j < 9; j++)
                        for (int k = 0; k < 4; k++) {
                            top_target[(size_t)(roi + j) * 4 * C + 4 * cls + k] = gp[6 + k];
                            top_weight[(size_t)(roi + j) * 4 * C + 4 * cls + k] = 1.f;
                        }
                    break;
                }
            }
        }
        const float x1 = b0[2], y1 = b0[3], x2 = b0[4], y2 = b0[5];
        const float ww = x2 - x1, hh = y2 - y1;
        // jitter order of .cu.cc:476-554; `x1 - 0.05 * ww` is double arithmetic
        const int jx[8] = {-1, 1, -1, 1, 0, -1, 0, 1};
        const int jy[8] = {-1, -1, 1, 1, -1, 0, 1, 0};
#pragma unroll
        for (int j = 0; j < 8; j++) {
            float* q = top_box + (size_t)(roi + 1 + j) * 7;
            q[0] = (float)(b + batch_offset);
            q[1] = (float)cls;
            q[2] = jx[j] == 0 ? x1 : (float)((double)x1 + jx[j] * (0.05 * (double)ww));
            q[3] = jy[j] == 0 ? y1 : (float)((double)y1 + jy[j] * (0.05 * (double)hh));
            q[4] = q[2] + ww;
            q[5] = q[3] + hh;
            q[6] = votes;
        }
    }
}

__global__ void k_zero2(float* a, size_t na, float* b, size_t nb)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, g = (size_t)gridDim.x * blockDim.x;
    for (size_t k = i; k < na / 4; k += g) reinterpret_cast<float4*>(a)[k] = make_float4(0, 0, 0, 0);
    for (size_t k = na / 4 * 4 + i; k < na; k += g) a[k] = 0.f;
    for (size_t k = i; k < nb / 4; k += g) reinterpret_cast<float4*>(b)[k] = make_float4(0, 0, 0, 0);
    for (size_t k = nb / 4 * 4 + i; k < nb; k += g) b[k] = 0.f;
}

// host side --------------------------------------------------------------------------------
static int run_front(const Layout& L, char* ws, const int32_t* label, const VertexSrc vertex, const float* extents,
                     const float* meta, int B, int H, int W, int C, int num_meta, float inlier, int label_thr, int skip,
                     ZeroList z, float* votes_out, cudaStream_t st)
{
    int* chunk_hist = (int*)(ws + L.chunk_hist);
    int* cls_size = (int*)(ws + L.cls_size);
    int* cls_slot = (int*)(ws + L.cls_slot);
    int* cls_nsamp = (int*)(ws + L.cls_nsamp);
    int* cls_soff = (int*)(ws + L.cls_soff);
    int* slot_cls = (int*)(ws + L.slot_cls);
    int* img_count = (int*)(ws + L.img_count);
    int* bbox = (int*)(ws + L.bbox);
    Sample* samples = (Sample*)(ws + L.samples);
    int2* band_res = (int2*)(ws + L.band_res);
    int* work = (int*)(ws + L.work);
    int* work_ctr = (int*)(ws + L.work_ctr);
    int* cand_n = (int*)(ws + L.cand_n);
    const int HW = H * W;
    dim3 grid(L.nchunks, B);
    cudaMemsetAsync(cls_size, 0, sizeof(int) * (size_t)B * C, st);
    k_hist<<<grid, kThreads, sizeof(int) * C, st>>>(label, HW, C, L.nchunks, chunk_hist, cls_size, bbox, cand_n, work_ctr, z);
    const size_t emit_smem = sizeof(int) * ((((kWarps + 7) * C + 1) & ~1) + 2 * kChunk);
    k_emit<<<grid, kThreads, emit_smem, st>>>(label, vertex, extents, meta, H, W, C, num_meta, L.nchunks, skip, label_thr,
                                              inlier, chunk_hist, cls_size, cls_slot, cls_nsamp, cls_soff, slot_cls,
                                              img_count, samples, L.samp_cap, bbox);
    k_worklist<<<1, 1024, 0, st>>>(B, C, L.R, L.nbands, img_count, slot_cls, cls_nsamp, bbox, work, work_ctr);
    size_t smem = sizeof(int) * (size_t)L.R * (W + 3);
    PCNN_SMEM_OPTIN(k_vote, 110 * 1024, "hough k_vote");
    // end points closer than tau0 (+ a term growing with the distance) to a cell centre are re-checked with the reference
    // predicate; the estimate's own error is ~1e-4 cells (DESIGN.md §3.3), the default keeps a 40x margin (0.438 -> 0.393 ms at batch 32
    // against 0.03, profiles/r02_hough_tau_sweep.txt); tests/test_hough_exact_gpu.py holds the planes to §3.3's exactness criterion
    static const float tau0 = getenv("PCNN_HOUGH_TAU0") ? (float)atof(getenv("PCNN_HOUGH_TAU0")) : 0.004f;
    k_vote<<<4 * kNumSMs, kThreads, smem, st>>>(H, W, C, L.R, L.nbands, inlier, tau0, slot_cls, cls_nsamp, cls_soff, bbox,
                                                samples, L.samp_cap, work, work_ctr, band_res, votes_out);
    return check_launch("hough front kernels");
}

static int validate(int B, int H, int W, int C, int skip)
{
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 2, "hough: need B,H,W >= 1 and C >= 2 (got %d,%d,%d,%d)", B, H, W, C);
    PCNN_REQUIRE(H <= 16383 && W <= 16383, "hough: image larger than 16383 x 16383 unsupported (got %d x %d)", W, H);
    PCNN_REQUIRE((long long)C * H * W < 0x7fffffffLL, "hough: C*H*W must fit int32 (reference flat index, .cu.cc:260)");
    PCNN_REQUIRE(skip >= 1, "hough: skip_pixels must be >= 1 (got %d)", skip);
    PCNN_REQUIRE(C <= 512, "hough: at most 512 classes supported (got %d)", C);
    return PCNN_OK;
}

}  // namespace hough
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::hough;

extern "C" int pcnn_hough_vote_workspace_bytes(int B, int H, int W, int C, int skip_pixels, float threshold_vote,
                                               size_t* bytes)
{
    int rc = validate(B, H, W, C, skip_pixels);
    if (rc) return rc;
    PCNN_REQUIRE(bytes != nullptr, "hough: bytes is NULL");
    const bool thr_mode = threshold_vote > 0;
    Layout L = make_layout(B, H, W, C, skip_pixels, /*want_votes=*/thr_mode, thr_mode);
    // + selection scratch of k_finalize
    *bytes = L.total + align_up(sizeof(int) * ((size_t)B * PCNN_MAX_ROI + B + 1), 256);
    return PCNN_OK;
}

static int hough_fwd_impl(const int32_t* label, const VertexSrc vsrc, const float* extents, const float* meta,
                          const float* gt, int B, int batch_global, int batch_offset, int H, int W, int C, int num_gt,
                          int num_meta, int is_train, float inlier_threshold, int label_threshold, float threshold_vote,
                          float threshold_percentage, int skip_pixels, float* top_box, float* top_pose,
                          float* top_target, float* top_weight, int32_t* top_domain, int32_t* num_rois,
                          int32_t* status, void* workspace, size_t workspace_bytes, void* stream)
{
    int rc = validate(B, H, W, C, skip_pixels);
    if (rc) return rc;
    PCNN_REQUIRE(is_train >= 0, "Need is_train >= 0, got %d", is_train);  // hough_voting_gpu_op.cc:309-311
    PCNN_REQUIRE(num_meta >= 6, "hough: meta_data needs the intrinsics (num_meta >= 6, got %d)", num_meta);
    PCNN_REQUIRE(num_gt == 0 || gt != nullptr, "hough: gt is NULL but num_gt = %d", num_gt);
    PCNN_REQUIRE(label && (vsrc.dense || (vsrc.lowres && vsrc.bias)) && extents && meta && top_box && top_pose &&
                     top_target && top_weight && top_domain && num_rois && workspace, "hough: NULL tensor pointer");
    PCNN_REQUIRE(batch_global >= B && batch_offset >= 0 && batch_offset + B <= batch_global,
                 "hough: shard [%d, %d) does not lie inside the global batch of %d images", batch_offset, batch_offset + B,
                 batch_global);
    const bool thr_mode = threshold_vote > 0;
    size_t need = 0;
    pcnn_hough_vote_workspace_bytes(B, H, W, C, skip_pixels, threshold_vote, &need);
    if (workspace_bytes < need) {
        set_error("hough: workspace too small (%zu < %zu)", workspace_bytes, need);
        return PCNN_E_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    Layout L = make_layout(B, H, W, C, skip_pixels, thr_mode, thr_mode);
    char* ws = (char*)workspace;
    int* sel = (int*)(ws + L.total);
    int* sel_n = sel + (size_t)B * PCNN_MAX_ROI;
    ZeroList z;
    const unsigned rows = PCNN_HOUGH_MAX_ROWS;
    z.p[0] = top_box; z.n[0] = rows * 7;
    z.p[1] = top_pose; z.n[1] = rows * 7;
    z.p[2] = top_target; z.n[2] = rows * 4 * C;
    z.p[3] = top_weight; z.n[3] = rows * 4 * C;
    z.p[4] = reinterpret_cast<float*>(top_domain); z.n[4] = rows;
    if (status) cudaMemsetAsync(status, 0, 4 * sizeof(int), st);
    float* votes = thr_mode ? (float*)(ws + L.votes) : nullptr;
    rc = run_front(L, ws, label, vsrc, extents, meta, B, H, W, C, num_meta, inlier_threshold, label_threshold,
                   skip_pixels, z, votes, st);
    if (rc) return rc;
    int* img_count = (int*)(ws + L.img_count);
    int* slot_cls = (int*)(ws + L.slot_cls);
    int* bbox = (int*)(ws + L.bbox);
    int* cand_key = (int*)(ws + L.cand_key);
    int* cand_val = (int*)(ws + L.cand_val);
    int* cand_n = (int*)(ws + L.cand_n);
    float4* cand_data = (float4*)(ws + L.cand_data);
    // .cu.cc:733: index_size = MAX_ROI / batch_size — of the WHOLE batch the reference op would see; a rank that
    // holds images [batch_offset, batch_offset + B) of it applies the same cap (SURVEY.md §8(e))
    const int cap = PCNN_MAX_ROI / batch_global;
    if (!thr_mode) {
        k_select<<<B, 32, 0, st>>>(C, H * W, L.R, L.nbands, cap, L.cand_cap, img_count, slot_cls, bbox,
                                   (const int2*)(ws + L.band_res), cand_key, cand_val, cand_n);
    } else {
        dim3 g((H * W + kThreads - 1) / kThreads, C - 1, B);
        k_localmax<<<g, kThreads, 0, st>>>(H, W, C, L.R, threshold_vote, L.cand_cap, img_count, slot_cls, bbox, votes,
                                           cand_key, cand_val, cand_n, status);
    }
    dim3 gcell(thr_mode ? 64 : (unsigned)std::max(1, std::min(std::min(cap, C), L.cand_cap)), B);
    k_celldata<<<gcell, kThreads, 0, st>>>(B, H, W, C, num_meta, inlier_threshold, L.cand_cap, extents, meta, slot_cls,
                                             (const int*)(ws + L.cls_nsamp), (const int*)(ws + L.cls_soff),
                                             (const Sample*)(ws + L.samples), L.samp_cap, cand_key, cand_n, cand_data);
    k_finalize<<<1, kThreads, 0, st>>>(B, batch_offset, H, W, C, num_meta, num_gt, is_train, cap, L.cand_cap,
                                       thr_mode ? 1 : 0, threshold_percentage, extents, meta, gt, slot_cls, cand_key, cand_val,
                                       cand_n, cand_data, sel, sel_n, top_box, top_pose, top_target, top_weight, top_domain,
                                       num_rois, status);
    return check_launch("hough back kernels");
}

extern "C" int pcnn_hough_vote_fwd(const int32_t* label, const float* vertex, const float* extents, const float* meta,
                                   const float* gt, int B, int H, int W, int C, int num_gt, int num_meta, int is_train,
                                   float inlier_threshold, int label_threshold, float threshold_vote,
                                   float threshold_percentage, int skip_pixels, float* top_box, float* top_pose,
                                   float* top_target, float* top_weight, int32_t* top_domain, int32_t* num_rois,
                                   int32_t* status, void* workspace, size_t workspace_bytes, void* stream)
{
    VertexSrc vs = {vertex, nullptr, nullptr, 0, 0};
    return hough_fwd_impl(label, vs, extents, meta, gt, B, B, 0, H, W, C, num_gt, num_meta, is_train, inlier_threshold,
                          label_threshold, threshold_vote, threshold_percentage, skip_pixels, top_box, top_pose, top_target,
                          top_weight, top_domain, num_rois, status, workspace, workspace_bytes, stream);
}

extern "C" int pcnn_hough_vote_fwd_ex(const int32_t* label, const float* vertex, const float* lowres,
                                      const float* bias_vertex, const float* extents, const float* meta, const float* gt,
                                      int B, int batch_global, int batch_offset, int H, int W, int C, int num_gt,
                                      int num_meta, int is_train, float inlier_threshold, int label_threshold,
                                      float threshold_vote, float threshold_percentage, int skip_pixels, float* top_box,
                                      float* top_pose, float* top_target, float* top_weight, int32_t* top_domain,
                                      int32_t* num_rois, int32_t* status, void* workspace, size_t workspace_bytes,
                                      void* stream)
{
    PCNN_REQUIRE(vertex || (H % 8 == 0 && W % 8 == 0), "hough: the lowres vertex source needs H, W multiples of 8 (got %d x %d)", H, W);
    VertexSrc vs = {vertex, vertex ? nullptr : lowres, vertex ? nullptr : bias_vertex, H / 8, W / 8};
    return hough_fwd_impl(label, vs, extents, meta, gt, B, batch_global, batch_offset, H, W, C, num_gt, num_meta, is_train,
                          inlier_threshold, label_threshold, threshold_vote, threshold_percentage, skip_pixels, top_box,
                          top_pose, top_target, top_weight, top_domain, num_rois, status, workspace, workspace_bytes, stream);
}

extern "C" int pcnn_hough_vote_planes(const int32_t* label, const float* vertex, const float* extents, const float* meta,
                                      int B, int H, int W, int C, int num_meta, float inlier_threshold,
                                      int label_threshold, int skip_pixels, float* votes, void* workspace,
                                      size_t workspace_bytes, void* stream)
{
    int rc = validate(B, H, W, C, skip_pixels);
    if (rc) return rc;
    PCNN_REQUIRE(label && vertex && extents && meta && votes && workspace, "hough planes: NULL tensor pointer");
    Layout L = make_layout(B, H, W, C, skip_pixels, false, false);
    if (workspace_bytes < L.total) {
        set_error("hough planes: workspace too small (%zu < %zu)", workspace_bytes, L.total);
        return PCNN_E_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(votes, 0, sizeof(float) * (size_t)B * C * H * W, st);
    ZeroList z;
    for (int k = 0; k < 5; k++) { z.p[k] = nullptr; z.n[k] = 0; }
    VertexSrc vs = {vertex, nullptr, nullptr, 0, 0};
    return run_front(L, (char*)workspace, label, vs, extents, meta, B, H, W, C, num_meta, inlier_threshold,
                     label_threshold, skip_pixels, z, votes, st);
}

extern "C" int pcnn_hough_vote_bwd(float* grad_label, float* grad_vertex, int B, int H, int W, int C, void* stream)
{
    PCNN_REQUIRE(grad_label && grad_vertex, "hough bwd: NULL pointer");
    size_t na = (size_t)B * H * W, nb = na * 3 * C;
    k_zero2<<<4 * kNumSMs, 256, 0, (cudaStream_t)stream>>>(grad_label, na, grad_vertex, nb);
    return check_launch("hough bwd");
}
