// pixel_ops.cu — RoiPool, Hardlabel, Project / Backproject and their gradients for sm_90a.
//
// All of these are HBM-bound gathers / streams (SURVEY.md §8(d)); the kernels keep the
// channel dimension (NHWC innermost) on adjacent lanes with 128-bit accesses, compute each
// geometric quantity once per (pixel|voxel|bin) group of lanes, and size grids from the
// element count (grid-stride loops, kNumSMs x resident CTAs).
//
// Behavioural specs (paths relative to /root/reference/lib):
//   RoiPool fwd/bwd  roi_pooling_layer/roi_pooling_op_gpu.cu.cc:19-101, 134-229
//   Hardlabel        hard_label_layer/hard_label_op_gpu.cu.cc:16-29, 54-63
//   Project          projecting_layer/projecting_op_gpu.cu.cc:16-73, 101-169
//   Backproject      backprojecting_layer/backprojecting_op_gpu.cu.cc:16-126, 158-217
#include <cuda_bf16.h>
#include <float.h>

#include <stdlib.h>

#include "common.cuh"

namespace pcnn {

static inline int grid_for(size_t work_items, int threads, int max_waves = 16)
{
    size_t blocks = (work_items + threads - 1) / threads;
    size_t cap = (size_t)kNumSMs * max_waves;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

// ----------------------------------------------------------------------------------------
// RoiPool forward: one thread per (roi, ph, pw, 4 channels)
// ----------------------------------------------------------------------------------------
struct RoiBin {
    int b, cls, hs, he, ws, we;
};

__device__ __forceinline__ RoiBin roi_bin(const float* __restrict__ r, int ph, int pw, int ph_n, int pw_n, float scale,
                                          int height, int width)
{
    RoiBin o;
    o.b = (int)r[0];
    o.cls = (int)r[1];
    int rsw = (int)roundf(__fmul_rn(r[2], scale)), rsh = (int)roundf(__fmul_rn(r[3], scale));
    int rew = (int)roundf(__fmul_rn(r[4], scale)), reh = (int)roundf(__fmul_rn(r[5], scale));
    int rw = max(rew - rsw + 1, 1), rh = max(reh - rsh + 1, 1);
    float bh = __fdiv_rn((float)rh, (float)ph_n), bw = __fdiv_rn((float)rw, (float)pw_n);
    int hs = (int)floorf(__fmul_rn((float)ph, bh)), wsx = (int)floorf(__fmul_rn((float)pw, bw));
    int he = (int)ceilf(__fmul_rn((float)(ph + 1), bh)), we = (int)ceilf(__fmul_rn((float)(pw + 1), bw));
    o.hs = min(max(hs + rsh, 0), height);
    o.he = min(max(he + rsh, 0), height);
    o.ws = min(max(wsx + rsw, 0), width);
    o.we = min(max(we + rsw, 0), width);
    return o;
}

template <int VEC>
__global__ void __launch_bounds__(256)
k_roi_pool_fwd(const float* __restrict__ bottom, const float* __restrict__ rois, int num_rois, int channel_rois, int batch,
               int height, int width, int channels, int ph_n, int pw_n, float scale, float* __restrict__ top,
               int* __restrict__ argmax)
{
    const int cg = channels / VEC;
    const size_t total = (size_t)num_rois * ph_n * pw_n * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        int g = (int)(idx % cg);
        size_t r1 = idx / cg;
        int pw = (int)(r1 % pw_n);
        r1 /= pw_n;
        int ph = (int)(r1 % ph_n);
        int n = (int)(r1 / ph_n);
        RoiBin rb = roi_bin(rois + (size_t)n * channel_rois, ph, pw, ph_n, pw_n, scale, height, width);
        bool empty = (rb.he <= rb.hs) || (rb.we <= rb.ws) || rb.b < 0 || rb.b >= batch;
        float mv[VEC];
        int mi[VEC];
#pragma unroll
        for (int k = 0; k < VEC; k++) { mv[k] = empty ? 0.f : -FLT_MAX; mi[k] = -1; }
        if (!empty) {
            const float* img = bottom + (size_t)rb.b * height * width * channels;
            for (int h = rb.hs; h < rb.he; h++)
                for (int w = rb.ws; w < rb.we; w++) {
                    int bi = (h * width + w) * channels + g * VEC;
                    float v[VEC];
                    if (VEC == 4) {
                        float4 q = __ldg(reinterpret_cast<const float4*>(img + bi));
                        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                    } else {
                        v[0] = __ldg(img + bi);
                    }
#pragma unroll
                    for (int k = 0; k < VEC; k++)
                        if (v[k] > mv[k]) { mv[k] = v[k]; mi[k] = bi + k; }
                }
        }
        size_t o = ((size_t)(n * ph_n + ph) * pw_n + pw) * channels + g * VEC;
        if (VEC == 4) {
            *reinterpret_cast<float4*>(top + o) = make_float4(mv[0], mv[1], mv[2], mv[3]);
            *reinterpret_cast<int4*>(argmax + o) = make_int4(mi[0], mi[1], mi[2], mi[3]);
        } else {
            top[o] = mv[0];
            argmax[o] = mi[0];
        }
    }
}

// same forward on bf16 NHWC features (the tensor-core trunk keeps activations in bf16): 8 channels per thread,
// fp32 outputs; comparisons are done on the bf16 values converted to fp32 (exact), so argmax is well defined
__global__ void __launch_bounds__(256)
k_roi_pool_fwd_bf16(const __nv_bfloat16* __restrict__ bottom, const float* __restrict__ rois, int num_rois, int channel_rois,
                    int batch, int height, int width, int channels, int ph_n, int pw_n, float scale, float* __restrict__ top,
                    int* __restrict__ argmax)
{
    const int cg = channels / 8;
    const size_t total = (size_t)num_rois * ph_n * pw_n * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        int g = (int)(idx % cg);
        size_t r1 = idx / cg;
        int pw = (int)(r1 % pw_n);
        r1 /= pw_n;
        int ph = (int)(r1 % ph_n);
        int n = (int)(r1 / ph_n);
        RoiBin rb = roi_bin(rois + (size_t)n * channel_rois, ph, pw, ph_n, pw_n, scale, height, width);
        bool empty = (rb.he <= rb.hs) || (rb.we <= rb.ws) || rb.b < 0 || rb.b >= batch;
        float mv[8];
        int mi[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { mv[k] = empty ? 0.f : -FLT_MAX; mi[k] = -1; }
        if (!empty) {
            const __nv_bfloat16* img = bottom + (size_t)rb.b * height * width * channels;
            for (int h = rb.hs; h < rb.he; h++)
#pragma unroll 4
                for (int w = rb.ws; w < rb.we; w++) {
                    int bi = (h * width + w) * channels + g * 8;
                    uint4 q = __ldg(reinterpret_cast<const uint4*>(img + bi));
                    const __nv_bfloat162* q2 = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        float2 f = __bfloat1622float2(q2[k]);
                        if (f.x > mv[2 * k]) { mv[2 * k] = f.x; mi[2 * k] = bi + 2 * k; }
                        if (f.y > mv[2 * k + 1]) { mv[2 * k + 1] = f.y; mi[2 * k + 1] = bi + 2 * k + 1; }
                    }
                }
        }
        size_t o = ((size_t)(n * ph_n + ph) * pw_n + pw) * channels + g * 8;
        *reinterpret_cast<float4*>(top + o) = make_float4(mv[0], mv[1], mv[2], mv[3]);
        *reinterpret_cast<float4*>(top + o + 4) = make_float4(mv[4], mv[5], mv[6], mv[7]);
        *reinterpret_cast<int4*>(argmax + o) = make_int4(mi[0], mi[1], mi[2], mi[3]);
        *reinterpret_cast<int4*>(argmax + o + 4) = make_int4(mi[4], mi[5], mi[6], mi[7]);
    }
}

// Sliced variant (channels % 32 == 0): the cells of a bin are dealt round-robin to 8 slices of 4 lanes (4 x 8 channels
// = 64 contiguous bytes of one pixel), four loads in flight per lane, and the (max, index) pairs are merged by
// shuffle -- "larger value, on ties the smaller index" reproduces the reference's raster-order scan with a strict '>'
// (.cu.cc:66-79).  A whole-image ROI has ~100 cells per bin at 1/8 resolution: the serial chain per lane is what
// bounded the one-thread-per-bin kernel (ncu: long-scoreboard 8.7 warps per issue).
constexpr int kRoiSlices = 8;
__global__ void __launch_bounds__(256)
k_roi_pool_fwd_bf16_s4(const __nv_bfloat16* __restrict__ bottom, const float* __restrict__ rois, int num_rois, int channel_rois,
                       int batch, int height, int width, int channels, int ph_n, int pw_n, float scale,
                       float* __restrict__ top, int* __restrict__ argmax)
{
    const int cgb = channels / 32;                                  // blocks of 4 channel groups (32 channels)
    const int lane = threadIdx.x & 31;
    const int gl = lane & 3, slice = lane >> 2;
    const int nwork = num_rois * ph_n * pw_n * cgb;                // one warp-task = (roi, bin, block of 32 channels)
    for (int task = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; task < nwork; task += (gridDim.x * blockDim.x) >> 5) {
        const int gb = task % cgb;
        int r1 = task / cgb;
        const int pw = r1 % pw_n; r1 /= pw_n;
        const int ph = r1 % ph_n;
        const int n = r1 / ph_n;
        const int ch0 = (gb * 4 + gl) * 8;
        RoiBin rb = roi_bin(rois + (size_t)n * channel_rois, ph, pw, ph_n, pw_n, scale, height, width);
        const bool empty = (rb.he <= rb.hs) || (rb.we <= rb.ws) || rb.b < 0 || rb.b >= batch;
        float mv[8];
        int mi[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { mv[k] = 0.f; mi[k] = -1; }
        if (!empty) {
            const __nv_bfloat16* img = bottom + (size_t)rb.b * height * width * channels;
            const int bw = rb.we - rb.ws, cells = bw * (rb.he - rb.hs);
            // Running maximum and its cell number stay PACKED: max as bf16x2 (HMNMX2), "is greater" as a 0xFFFF-per-half
            // mask (HSET2), cell number as u16x2 merged with one LOP3 -- 3 instructions per channel pair and cell instead
            // of 8 on unpacked floats.  Cell number = position in the bin's raster scan (< 65536: a bin has at most
            // height * width cells, checked on the host), so "smaller cell number" == "earlier in the reference's scan".
            // Start value -inf: every finite feature is greater, like the reference's -FLT_MAX (.cu.cc:57).
            uint32_t m2[4], c2[4];
#pragma unroll
            for (int k = 0; k < 4; k++) { m2[k] = 0xff80ff80u; c2[k] = 0xffffffffu; }
            for (int i0 = slice; i0 < cells; i0 += 4 * kRoiSlices) {
                uint4 q[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int ic = min(i0 + u * kRoiSlices, cells - 1);
                    const int hh = ic / bw, ww = ic - hh * bw;
                    q[u] = __ldg(reinterpret_cast<const uint4*>(img + ((rb.hs + hh) * width + rb.ws + ww) * channels + ch0));
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int i = i0 + u * kRoiSlices;
                    if (i >= cells) continue;
                    const uint32_t i2 = (uint32_t)i * 0x10001u;
                    const uint32_t* qw = reinterpret_cast<const uint32_t*>(&q[u]);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&qw[k]);
                        const __nv_bfloat162 m = *reinterpret_cast<const __nv_bfloat162*>(&m2[k]);
                        const uint32_t gt = __hgt2_mask(v, m);              // strict '>' per half (.cu.cc:73)
                        const __nv_bfloat162 nm = __hmax2(v, m);
                        m2[k] = *reinterpret_cast<const uint32_t*>(&nm);
                        c2[k] = (c2[k] & ~gt) | (i2 & gt);
                    }
                }
            }
            // merge the slices: larger value, on ties the smaller cell number (a slice without cells holds -inf / 0xffff)
#pragma unroll
            for (int d = 4; d <= 16; d <<= 1) {
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const uint32_t om = __shfl_xor_sync(0xffffffffu, m2[k], d);
                    const uint32_t oc = __shfl_xor_sync(0xffffffffu, c2[k], d);
                    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&m2[k]);
                    const __nv_bfloat162 o = *reinterpret_cast<const __nv_bfloat162*>(&om);
                    const uint32_t gt = __hgt2_mask(o, a), eq = __heq2_mask(o, a);
                    // per half: other cell number smaller?  (16-bit unsigned compare on both halves)
                    const uint32_t lo_lt = ((oc & 0xffffu) < (c2[k] & 0xffffu)) ? 0x0000ffffu : 0u;
                    const uint32_t hi_lt = ((oc >> 16) < (c2[k] >> 16)) ? 0xffff0000u : 0u;
                    const uint32_t take = gt | (eq & (lo_lt | hi_lt));
                    m2[k] = (m2[k] & ~take) | (om & take);
                    c2[k] = (c2[k] & ~take) | (oc & take);
                }
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&m2[k]));
                const int i_lo = (int)(c2[k] & 0xffffu), i_hi = (int)(c2[k] >> 16);
                // every non-empty bin has at least one cell and all features are finite -> a cell number was recorded;
                // 0xffff survives only if the feature was -inf / NaN, reported like the reference's untouched start value
                mv[2 * k] = i_lo == 0xffff ? -FLT_MAX : f.x;
                mv[2 * k + 1] = i_hi == 0xffff ? -FLT_MAX : f.y;
                const int h_lo = i_lo / bw, h_hi = i_hi / bw;
                mi[2 * k] = i_lo == 0xffff ? -1 : ((rb.hs + h_lo) * width + rb.ws + (i_lo - h_lo * bw)) * channels + ch0 + 2 * k;
                mi[2 * k + 1] = i_hi == 0xffff ? -1 : ((rb.hs + h_hi) * width + rb.ws + (i_hi - h_hi * bw)) * channels + ch0 + 2 * k + 1;
            }
        }
        if (slice == 0) {
            const size_t o = ((size_t)(n * ph_n + ph) * pw_n + pw) * channels + ch0;
            *reinterpret_cast<float4*>(top + o) = make_float4(mv[0], mv[1], mv[2], mv[3]);
            *reinterpret_cast<float4*>(top + o + 4) = make_float4(mv[4], mv[5], mv[6], mv[7]);
            *reinterpret_cast<int4*>(argmax + o) = make_int4(mi[0], mi[1], mi[2], mi[3]);
            *reinterpret_cast<int4*>(argmax + o + 4) = make_int4(mi[4], mi[5], mi[6], mi[7]);
        }
    }
}

// pool_channel mode: one output channel = channel roi_cls of the input (.cu.cc:84-87)
__global__ void __launch_bounds__(256)
k_roi_pool_fwd_cls(const float* __restrict__ bottom, const float* __restrict__ rois, int num_rois, int channel_rois,
                   int batch, int height, int width, int channels, int ph_n, int pw_n, float scale,
                   float* __restrict__ top, int* __restrict__ argmax)
{
    const int total = num_rois * ph_n * pw_n;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        int pw = idx % pw_n, ph = (idx / pw_n) % ph_n, n = idx / (pw_n * ph_n);
        RoiBin rb = roi_bin(rois + (size_t)n * channel_rois, ph, pw, ph_n, pw_n, scale, height, width);
        bool empty = (rb.he <= rb.hs) || (rb.we <= rb.ws) || rb.b < 0 || rb.b >= batch || rb.cls < 0 || rb.cls >= channels;
        float mv = empty ? 0.f : -FLT_MAX;
        int mi = -1;
        if (!empty) {
            const float* img = bottom + (size_t)rb.b * height * width * channels;
            for (int h = rb.hs; h < rb.he; h++)
                for (int w = rb.ws; w < rb.we; w++) {
                    int bi = (h * width + w) * channels + rb.cls;
                    float v = __ldg(img + bi);
                    if (v > mv) { mv = v; mi = bi; }
                }
        }
        top[idx] = mv;
        argmax[idx] = mi;
    }
}

// RoiPool backward as a scatter through argmax: grad_in[b, argmax] += top_diff.  The
// reference gathers per input element over ALL rois (.cu.cc:153) and accepts a (bin, element)
// pair iff the element lies inside the un-clipped roi (.cu.cc:176-181), the bin lies in the
// element's feasible bin range (.cu.cc:203-211) and the bin's argmax is that element; the
// same three tests are applied here per pooled value, so the set of contributions is identical
// (malformed rois, whose forward is forced to 1x1, contribute nothing — as in the reference).
struct RoiGeom {
    int b, rsw, rsh, rew, reh;
    float bh, bw;
};

__device__ __forceinline__ RoiGeom roi_geom(const float* __restrict__ r, float scale, int ph_n, int pw_n)
{
    RoiGeom g;
    g.b = (int)r[0];
    g.rsw = (int)roundf(__fmul_rn(r[2], scale)); g.rsh = (int)roundf(__fmul_rn(r[3], scale));
    g.rew = (int)roundf(__fmul_rn(r[4], scale)); g.reh = (int)roundf(__fmul_rn(r[5], scale));
    int rw = max(g.rew - g.rsw + 1, 1), rh = max(g.reh - g.rsh + 1, 1);
    g.bh = __fdiv_rn((float)rh, (float)ph_n);
    g.bw = __fdiv_rn((float)rw, (float)pw_n);
    return g;
}

__device__ __forceinline__ bool roi_bwd_accepts(const RoiGeom& g, int a, int width, int channels, int ph, int pw, int ph_n,
                                                int pw_n)
{
    int pix = a / channels;
    int h = pix / width, w = pix % width;
    if (!(w >= g.rsw && w <= g.rew && h >= g.rsh && h <= g.reh)) return false;
    int phs = (int)floorf(__fdiv_rn((float)(h - g.rsh), g.bh)), phe = (int)ceilf(__fdiv_rn((float)(h - g.rsh + 1), g.bh));
    int pws = (int)floorf(__fdiv_rn((float)(w - g.rsw), g.bw)), pwe = (int)ceilf(__fdiv_rn((float)(w - g.rsw + 1), g.bw));
    phs = min(max(phs, 0), ph_n); phe = min(max(phe, 0), ph_n);
    pws = min(max(pws, 0), pw_n); pwe = min(max(pwe, 0), pw_n);
    return ph >= phs && ph < phe && pw >= pws && pw < pwe;
}

template <int VEC>
__global__ void __launch_bounds__(256)
k_roi_pool_bwd(const float* __restrict__ top_diff, const int* __restrict__ argmax, const float* __restrict__ rois,
               int batch, int num_rois, int channel_rois, int height, int width, int channels, int out_ch, int ph_n,
               int pw_n, float scale, float* __restrict__ bottom_diff)
{
    const int cg = out_ch / VEC;
    const int bins = ph_n * pw_n;
    const size_t total = (size_t)num_rois * bins * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        size_t e = idx * VEC;
        int n = (int)(e / ((size_t)bins * out_ch));
        int bin = (int)((e / out_ch) % bins);
        int ph = bin / pw_n, pw = bin % pw_n;
        RoiGeom g = roi_geom(rois + (size_t)n * channel_rois, scale, ph_n, pw_n);
        if (g.b < 0 || g.b >= batch) continue;
        float* img = bottom_diff + (size_t)g.b * height * width * channels;
        int a[VEC];
        float d[VEC];
        if (VEC == 4) {
            int4 av = *reinterpret_cast<const int4*>(argmax + e);
            float4 dv = *reinterpret_cast<const float4*>(top_diff + e);
            a[0] = av.x; a[1] = av.y; a[2] = av.z; a[3] = av.w;
            d[0] = dv.x; d[1] = dv.y; d[2] = dv.z; d[3] = dv.w;
        } else {
            a[0] = argmax[e];
            d[0] = top_diff[e];
        }
#pragma unroll
        for (int k = 0; k < VEC; k++)
            if (a[k] >= 0 && roi_bwd_accepts(g, a[k], width, channels, ph, pw, ph_n, pw_n)) atomicAdd(img + a[k], d[k]);
    }
}

__global__ void __launch_bounds__(256) k_fill_zero(float* __restrict__ p, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, g = (size_t)gridDim.x * blockDim.x;
    size_t n4 = n / 4;
    for (size_t k = i; k < n4; k += g) st_stream_f4(reinterpret_cast<float4*>(p) + k, make_float4(0, 0, 0, 0));
    for (size_t k = n4 * 4 + i; k < n; k += g) p[k] = 0.f;
}

// ----------------------------------------------------------------------------------------
// Hardlabel: streaming one-hot writer.  out[p,:] = 0; out[p,g] = 1 iff g != -1 and
// (g > 0 or prob[p,g] < threshold).  Labels outside [-1, C) write nothing (the reference
// would write out of bounds there).
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_hard_label(const float* __restrict__ prob, const int* __restrict__ gt, size_t npix, int C, float threshold,
             float* __restrict__ top)
{
    const size_t total = npix * C;
    const size_t n4 = total / 4;
    const size_t g0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, gs = (size_t)gridDim.x * blockDim.x;
    for (size_t k = g0; k < n4; k += gs) {
        size_t e = k * 4;
        size_t p = e / C;
        int ch = (int)(e % C);
        float v[4];
        int g = gt[p];
        bool hot = g >= 0 && g < C && (g > 0 || __ldg(prob + p * C) < threshold);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            v[j] = (hot && ch == g) ? 1.f : 0.f;
            if (++ch == C) {
                ch = 0;
                p++;
                if (j < 3 && p < npix) {
                    g = gt[p];
                    hot = g >= 0 && g < C && (g > 0 || __ldg(prob + p * C) < threshold);
                }
            }
        }
        st_stream_f4(reinterpret_cast<float4*>(top) + k, make_float4(v[0], v[1], v[2], v[3]));
    }
    for (size_t e = n4 * 4 + g0; e < total; e += gs) {
        size_t p = e / C;
        int ch = (int)(e % C);
        int g = gt[p];
        bool hot = g >= 0 && g < C && (g > 0 || prob[p * C] < threshold);
        top[e] = (hot && ch == g) ? 1.f : 0.f;
    }
}

// ----------------------------------------------------------------------------------------
// Project / Backproject geometry (same rounding as nvcc gives the reference expressions)
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ bool pixel_to_voxel(const float* __restrict__ m, int w, int h, float depth, int G, int& vd,
                                               int& vh, int& vw)
{
    float fw = (float)w, fh = (float)h;
    float RX = __fadd_rn(__fmaf_rn(m[9], fw, __fmul_rn(m[10], fh)), m[11]);
    float RY = __fadd_rn(__fmaf_rn(m[12], fw, __fmul_rn(m[13], fh)), m[14]);
    float RZ = __fadd_rn(__fmaf_rn(m[15], fw, __fmul_rn(m[16], fh)), m[17]);
    float X = __fmul_rn(depth, RX), Y = __fmul_rn(depth, RY), Z = __fmul_rn(depth, RZ);
    float X1 = __fadd_rn(__fmaf_rn(m[32], Z, __fmaf_rn(m[30], X, __fmul_rn(m[31], Y))), m[33]);
    float Y1 = __fadd_rn(__fmaf_rn(m[36], Z, __fmaf_rn(m[34], X, __fmul_rn(m[35], Y))), m[37]);
    float Z1 = __fadd_rn(__fmaf_rn(m[40], Z, __fmaf_rn(m[38], X, __fmul_rn(m[39], Y))), m[41]);
    vd = (int)roundf(__fdiv_rn(__fsub_rn(X1, m[45]), m[42]));
    vh = (int)roundf(__fdiv_rn(__fsub_rn(Y1, m[46]), m[43]));
    vw = (int)roundf(__fdiv_rn(__fsub_rn(Z1, m[47]), m[44]));
    return vd >= 0 && vd < G && vh >= 0 && vh < G && vw >= 0 && vw < G;
}

__device__ __forceinline__ void voxel_to_pixel(const float* __restrict__ m, int d, int h, int w, int& px, int& py,
                                               float& Z1)
{
    float X = __fmaf_rn((float)d, m[42], m[45]);
    float Y = __fmaf_rn((float)h, m[43], m[46]);
    float Z = __fmaf_rn((float)w, m[44], m[47]);
    float X1 = __fadd_rn(__fmaf_rn(m[20], Z, __fmaf_rn(m[18], X, __fmul_rn(m[19], Y))), m[21]);
    float Y1 = __fadd_rn(__fmaf_rn(m[24], Z, __fmaf_rn(m[22], X, __fmul_rn(m[23], Y))), m[25]);
    Z1 = __fadd_rn(__fmaf_rn(m[28], Z, __fmaf_rn(m[26], X, __fmul_rn(m[27], Y))), m[29]);
    float x1 = __fmaf_rn(m[2], Z1, __fmaf_rn(m[0], X1, __fmul_rn(m[1], Y1)));
    float x2 = __fmaf_rn(m[5], Z1, __fmaf_rn(m[3], X1, __fmul_rn(m[4], Y1)));
    float x3 = __fmaf_rn(m[8], Z1, __fmaf_rn(m[6], X1, __fmul_rn(m[7], Y1)));
    float a = __fdiv_rn(x1, x3), b = __fdiv_rn(x2, x3);
    // clamp before the int conversion so that inf / NaN cannot produce a bogus in-range pixel
    a = fminf(fmaxf(a, -1e8f), 1e8f);
    b = fminf(fmaxf(b, -1e8f), 1e8f);
    px = (a == a) ? (int)roundf(a) : -0x40000000;
    py = (b == b) ? (int)roundf(b) : -0x40000000;
}

// out[B,H,W,Cf] = vox[B,G,G,G,Cf] at the voxel hit by each pixel, else 0
// (ProjectForward .cu.cc:16-73; BackprojectBackward .cu.cc:158-217)
template <int VEC>
__global__ void __launch_bounds__(256)
k_pixel_gather(const float* __restrict__ vox, const float* __restrict__ depth, const float* __restrict__ meta, int B,
               int H, int W, int Cf, int num_meta, int G, float* __restrict__ out)
{
    // grid.y = image; 32-bit index math inside the image (64-bit div/mod costs ~100 instructions each)
    const unsigned cg = Cf / VEC;
    const unsigned total = (unsigned)H * W * cg;
    const int n = blockIdx.y;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int g = (int)(i % cg);
        const unsigned pl = i / cg;
        const int w = (int)(pl % W), h = (int)(pl / W);
        const size_t pix = (size_t)n * H * W + pl;
        int vd, vh, vw;
        bool inside = pixel_to_voxel(meta + (size_t)n * num_meta, w, h, __ldg(depth + pix), G, vd, vh, vw);
        if (VEC == 4) {
            float4 v = make_float4(0, 0, 0, 0);
            if (inside) v = __ldg(reinterpret_cast<const float4*>(vox + ((((size_t)n * G + vd) * G + vh) * G + vw) * Cf) + g);
            st_stream_f4(reinterpret_cast<float4*>(out + pix * Cf) + g, v);
        } else {
            out[pix * Cf + g] = inside ? __ldg(vox + ((((size_t)n * G + vd) * G + vh) * G + vw) * Cf + g) : 0.f;
        }
    }
}

// window average of a [B,H,W,nch] map into a [B,G,G,G,nch] grid
// (BackprojectForward .cu.cc:16-126 for data (+flag) and labels (+label_3d fallback);
//  ProjectBackward .cu.cc:101-169 for top_diff)
template <int VEC>
__global__ void __launch_bounds__(256)
k_voxel_average(const float* __restrict__ src, const float* __restrict__ depth, const float* __restrict__ meta,
                const float* __restrict__ fallback, int B, int H, int W, int nch, int num_meta, int G, int ks,
                float threshold, float* __restrict__ dst, float* __restrict__ flag)
{
    // grid.y = image; 32-bit index math inside the image
    const unsigned cg = nch / VEC;
    const unsigned total = (unsigned)G * G * G * cg;
    const int n = blockIdx.y;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int g = (int)(i % cg);
        const unsigned vl = i / cg;
        const int w = (int)(vl % G), h = (int)((vl / G) % G), d = (int)(vl / ((unsigned)G * G));
        const size_t vox = (size_t)n * G * G * G + vl;
        int px, py;
        float Z1;
        voxel_to_pixel(meta + (size_t)n * num_meta, d, h, w, px, py, Z1);
        float acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; k++) acc[k] = 0.f;
        int count = 0;
        const int x0 = max(px - ks, 0), x1 = min(px + ks, W - 1);
        const int y0 = max(py - ks, 0), y1 = min(py + ks, H - 1);
        for (int x = x0; x <= x1; x++)
            for (int y = y0; y <= y1; y++) {
                size_t pix = ((size_t)n * H + y) * W + x;
                float dep = __ldg(depth + pix);
                if (fabsf(__fsub_rn(dep, Z1)) < threshold) {
                    count++;
                    if (VEC == 4) {
                        float4 q = __ldg(reinterpret_cast<const float4*>(src + pix * nch) + g);
                        acc[0] += q.x; acc[1] += q.y; acc[2] += q.z; acc[3] += q.w;
                    } else {
                        acc[0] += __ldg(src + pix * nch + g);
                    }
                }
            }
        float fl = 0.f;
        if (count == 0) {
            if (fallback) {
                if (VEC == 4) {
                    float4 q = __ldg(reinterpret_cast<const float4*>(fallback + vox * nch) + g);
                    acc[0] = q.x; acc[1] = q.y; acc[2] = q.z; acc[3] = q.w;
                } else {
                    acc[0] = __ldg(fallback + vox * nch + g);
                }
            }
        } else {
            float cf = (float)count;
#pragma unroll
            for (int k = 0; k < VEC; k++) acc[k] = __fdiv_rn(acc[k], cf);
            fl = 1.f;
        }
        if (VEC == 4) {
            st_stream_f4(reinterpret_cast<float4*>(dst + vox * nch) + g, make_float4(acc[0], acc[1], acc[2], acc[3]));
            if (flag) st_stream_f4(reinterpret_cast<float4*>(flag + vox * nch) + g, make_float4(fl, fl, fl, fl));
        } else {
            dst[vox * nch + g] = acc[0];
            if (flag) flag[vox * nch + g] = fl;
        }
    }
}

// Wide-thread forms of the window average: every thread of k_voxel_average repeats the (2k+1)^2 depth tests of its
// voxel, so fewer threads per voxel = fewer redundant tests.  CPT channels per thread, kept in registers:
//   CPT = 16 (nch % 16 == 0): four 128-bit loads per hit, four streaming stores;
//   CPT = 32 (nch <= 32, e.g. the C = 22 label channels): one thread owns the whole voxel.
template <int CPT, bool WHOLE>
__global__ void __launch_bounds__(256)
k_voxel_average_wide(const float* __restrict__ src, const float* __restrict__ depth, const float* __restrict__ meta,
                     const float* __restrict__ fallback, int H, int W, int nch, int num_meta, int G, int ks,
                     float threshold, float* __restrict__ dst, float* __restrict__ flag)
{
    const unsigned cg = WHOLE ? 1u : (unsigned)nch / CPT;
    const unsigned total = (unsigned)G * G * G * cg;
    const int n = blockIdx.y;
    const int nc = WHOLE ? nch : CPT;  // channels handled by this thread
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int g = (int)(i % cg);
        const unsigned vl = i / cg;
        const int w = (int)(vl % G), h = (int)((vl / G) % G), d = (int)(vl / ((unsigned)G * G));
        const size_t vox = (size_t)n * G * G * G + vl;
        int px, py;
        float Z1;
        voxel_to_pixel(meta + (size_t)n * num_meta, d, h, w, px, py, Z1);
        float acc[CPT];
#pragma unroll
        for (int k = 0; k < CPT; k++) acc[k] = 0.f;
        int count = 0;
        const int x0 = max(px - ks, 0), x1 = min(px + ks, W - 1);
        const int y0 = max(py - ks, 0), y1 = min(py + ks, H - 1);
        for (int x = x0; x <= x1; x++)
            for (int y = y0; y <= y1; y++) {
                const size_t pix = ((size_t)n * H + y) * W + x;
                if (fabsf(__fsub_rn(__ldg(depth + pix), Z1)) < threshold) {
                    count++;
                    const float* sp = src + pix * nch + g * CPT;
                    if (!WHOLE) {
#pragma unroll
                        for (int k = 0; k < CPT; k += 4) {
                            const float4 q = __ldg(reinterpret_cast<const float4*>(sp + k));
                            acc[k] += q.x; acc[k + 1] += q.y; acc[k + 2] += q.z; acc[k + 3] += q.w;
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < CPT; k++)
                            if (k < nc) acc[k] += __ldg(sp + k);
                    }
                }
            }
        float fl = 0.f;
        if (count == 0) {
            if (fallback) {
                const float* fp = fallback + vox * nch + g * CPT;
#pragma unroll
                for (int k = 0; k < CPT; k++)
                    if (k < nc) acc[k] = __ldg(fp + k);
            }
        } else {
            const float cf = (float)count;
#pragma unroll
            for (int k = 0; k < CPT; k++) acc[k] = __fdiv_rn(acc[k], cf);
            fl = 1.f;
        }
        float* dp = dst + vox * nch + g * CPT;
        if (!WHOLE) {
#pragma unroll
            for (int k = 0; k < CPT; k += 4) {
                st_stream_f4(reinterpret_cast<float4*>(dp + k), make_float4(acc[k], acc[k + 1], acc[k + 2], acc[k + 3]));
                if (flag) st_stream_f4(reinterpret_cast<float4*>(flag + vox * nch + g * CPT + k), make_float4(fl, fl, fl, fl));
            }
        } else {
#pragma unroll
            for (int k = 0; k < CPT; k++)
                if (k < nc) { dp[k] = acc[k]; if (flag) flag[vox * nch + k] = fl; }
        }
    }
}

// ----------------------------------------------------------------------------------------
// BackprojectForward fused (backprojecting_op_gpu.cu.cc:16-126): ONE kernel writes top_data, top_flag and top_label.
// A CTA owns a slab of kBpVox consecutive voxels of one image:
//   phase 1  one thread per voxel: voxel -> pixel projection and the (2k+1)^2 depth tests ONCE per voxel (the separate
//            data / label launches with one thread per 16 channels repeated them 5 times); count, (px, py, Z1) -> smem;
//   phase 2  all threads stream the slab's three contiguous output regions with 128-bit stores (data: Cf floats per
//            voxel, flag likewise, label: C floats per voxel): voxels without a hit (almost all of the grid) are pure
//            stores — zeros, zeros, and the label_3d copy; the few voxels with hits re-walk their window in the
//            reference's order (x outer, y inner) and average.
// The op is write-bound: B * G^3 * (2 Cf + C) * 4 bytes out, B * G^3 * C * 4 + the touched pixels in.
// ----------------------------------------------------------------------------------------
constexpr int kBpVox = 64;

__global__ void __launch_bounds__(256)
k_backproject_fused(const float* __restrict__ data, const float* __restrict__ label, const float* __restrict__ depth,
                    const float* __restrict__ meta_all, const float* __restrict__ label_3d, int H, int W, int Cf, int C, int num_meta,
                    int G, int ks, float threshold, float* __restrict__ top_data, float* __restrict__ top_label,
                    float* __restrict__ top_flag)
{
    __shared__ int s_cnt[kBpVox], s_px[kBpVox], s_py[kBpVox];
    __shared__ float s_z[kBpVox];
    const int n = blockIdx.y, t = threadIdx.x;
    const unsigned G3 = (unsigned)G * G * G;
    const unsigned v0 = blockIdx.x * kBpVox;
    const int nvox = (int)min((unsigned)kBpVox, G3 - v0);
    const float* m = meta_all + (size_t)n * num_meta;
    const float* dep = depth + (size_t)n * H * W;
    if (t < nvox) {
        const unsigned vl = v0 + t;
        const int w = (int)(vl % G), h = (int)((vl / G) % G), d = (int)(vl / ((unsigned)G * G));
        int px, py;
        float Z1;
        voxel_to_pixel(m, d, h, w, px, py, Z1);
        int count = 0;
        const int x0 = max(px - ks, 0), x1 = min(px + ks, W - 1);
        const int y0 = max(py - ks, 0), y1 = min(py + ks, H - 1);
        for (int x = x0; x <= x1; x++)
            for (int y = y0; y <= y1; y++)
                if (fabsf(__fsub_rn(__ldg(dep + (size_t)y * W + x), Z1)) < threshold) count++;
        s_cnt[t] = count; s_px[t] = px; s_py[t] = py; s_z[t] = Z1;
    }
    __syncthreads();
    const size_t vbase = (size_t)n * G3 + v0;
    // ---- top_data / top_flag: Cf / 4 float4 per voxel
    {
        const int q4 = Cf >> 2;
        float4* od = reinterpret_cast<float4*>(top_data + vbase * Cf);
        float4* of = reinterpret_cast<float4*>(top_flag + vbase * Cf);
        const float* src = data + (size_t)n * H * W * Cf;
        for (int i = t; i < nvox * q4; i += 256) {
            const int v = i / q4, g = i - v * q4;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float fl = 0.f;
            const int cnt = s_cnt[v];
            if (cnt > 0) {
                const int px = s_px[v], py = s_py[v];
                const float Z1 = s_z[v];
                const int x0 = max(px - ks, 0), x1 = min(px + ks, W - 1);
                const int y0 = max(py - ks, 0), y1 = min(py + ks, H - 1);
                for (int x = x0; x <= x1; x++)
                    for (int y = y0; y <= y1; y++) {
                        const size_t pix = (size_t)y * W + x;
                        if (fabsf(__fsub_rn(__ldg(dep + pix), Z1)) < threshold) {
                            const float4 q = __ldg(reinterpret_cast<const float4*>(src + pix * Cf) + g);
                            acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
                        }
                    }
                const float cf = (float)cnt;
                acc.x = __fdiv_rn(acc.x, cf); acc.y = __fdiv_rn(acc.y, cf); acc.z = __fdiv_rn(acc.z, cf); acc.w = __fdiv_rn(acc.w, cf);
                fl = 1.f;
            }
            st_stream_f4(od + i, acc);
            st_stream_f4(of + i, make_float4(fl, fl, fl, fl));
        }
    }
    // ---- top_label: C floats per voxel; the slab's nvox * C floats are contiguous (float4 path when the slab is 16-byte
    // aligned and whole: kBpVox * C * 4 bytes is a multiple of 16 for every C).  The float4 path decides per group of 4
    // elements from the voxels of its first and last element, which are all the voxels the group touches only for C >= 2;
    // with C = 1 the group spans four voxels, so C = 1 takes the per-element path.
    {
        float* ol = top_label + vbase * C;
        const float* l3 = label_3d + vbase * C;
        const float* src = label + (size_t)n * H * W * C;
        const int total = nvox * C;
        auto element = [&](int i) -> float {
            const int v = i / C, c = i - v * C;
            const int cnt = s_cnt[v];
            if (cnt == 0) return __ldg(l3 + i);
            const int px = s_px[v], py = s_py[v];
            const float Z1 = s_z[v];
            const int x0 = max(px - ks, 0), x1 = min(px + ks, W - 1);
            const int y0 = max(py - ks, 0), y1 = min(py + ks, H - 1);
            float acc = 0.f;
            for (int x = x0; x <= x1; x++)
                for (int y = y0; y <= y1; y++) {
                    const size_t pix = (size_t)y * W + x;
                    if (fabsf(__fsub_rn(__ldg(dep + pix), Z1)) < threshold) acc += __ldg(src + pix * C + c);
                }
            return __fdiv_rn(acc, (float)cnt);
        };
        if (C > 1 && (total & 3) == 0 && ((reinterpret_cast<uintptr_t>(ol) | reinterpret_cast<uintptr_t>(l3)) & 15) == 0) {
            for (int i4 = t; i4 < total / 4; i4 += 256) {
                const int i = 4 * i4;
                const int va = i / C, vb = (i + 3) / C;
                float4 o;
                if (s_cnt[va] == 0 && s_cnt[vb] == 0) o = ld_stream_f4(reinterpret_cast<const float4*>(l3) + i4);
                else o = make_float4(element(i), element(i + 1), element(i + 2), element(i + 3));
                st_stream_f4(reinterpret_cast<float4*>(ol) + i4, o);
            }
        } else {
            for (int i = t; i < total; i += 256) ol[i] = element(i);
        }
    }
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace pcnn

using namespace pcnn;

extern "C" int pcnn_roi_pool_fwd(const float* bottom, const float* rois, int num_rois, int channel_rois, int batch,
                                 int height, int width, int channels, int pooled_height, int pooled_width,
                                 float spatial_scale, int pool_channel, float* top, int32_t* argmax, void* stream)
{
    PCNN_REQUIRE(pooled_height >= 0, "Need pooled_height >= 0, got %d", pooled_height);  // roi_pooling_op.cc:286-288
    PCNN_REQUIRE(pooled_width >= 0, "Need pooled_width >= 0, got %d", pooled_width);
    PCNN_REQUIRE(channel_rois >= 6, "rois must have at least 6 columns [b, cls, x1, y1, x2, y2] (got %d)", channel_rois);
    PCNN_REQUIRE(num_rois >= 0 && batch >= 1 && height >= 1 && width >= 1 && channels >= 1, "roi_pool: bad shape");
    PCNN_REQUIRE(bottom && rois && top && argmax, "roi_pool: NULL tensor pointer");
    if (num_rois == 0 || pooled_height == 0 || pooled_width == 0) return PCNN_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (pool_channel) {
        int total = num_rois * pooled_height * pooled_width;
        k_roi_pool_fwd_cls<<<grid_for(total, 256), 256, 0, st>>>(bottom, rois, num_rois, channel_rois, batch, height, width,
                                                                 channels, pooled_height, pooled_width, spatial_scale, top,
                                                                 argmax);
    } else if (channels % 4 == 0 && aligned16(bottom) && aligned16(top) && aligned16(argmax)) {
        size_t total = (size_t)num_rois * pooled_height * pooled_width * (channels / 4);
        k_roi_pool_fwd<4><<<grid_for(total, 256), 256, 0, st>>>(bottom, rois, num_rois, channel_rois, batch, height, width,
                                                                channels, pooled_height, pooled_width, spatial_scale, top,
                                                                argmax);
    } else {
        size_t total = (size_t)num_rois * pooled_height * pooled_width * channels;
        k_roi_pool_fwd<1><<<grid_for(total, 256), 256, 0, st>>>(bottom, rois, num_rois, channel_rois, batch, height, width,
                                                                channels, pooled_height, pooled_width, spatial_scale, top,
                                                                argmax);
    }
    return check_launch("roi_pool_fwd");
}

extern "C" int pcnn_roi_pool_bwd(const float* top_diff, const int32_t* argmax, const float* rois, int batch,
                                 int num_rois, int channel_rois, int height, int width, int channels,
                                 int pooled_height, int pooled_width, float spatial_scale, int pool_channel,
                                 float* bottom_diff, void* stream)
{
    PCNN_REQUIRE(channel_rois >= 6, "rois must have at least 6 columns (got %d)", channel_rois);
    PCNN_REQUIRE(top_diff && argmax && rois && bottom_diff, "roi_pool_grad: NULL tensor pointer");
    PCNN_REQUIRE(batch >= 1 && height >= 1 && width >= 1 && channels >= 1 && num_rois >= 0, "roi_pool_grad: bad shape");
    cudaStream_t st = (cudaStream_t)stream;
    size_t n_in = (size_t)batch * height * width * channels;
    k_fill_zero<<<grid_for(n_in / 4 + 1, 256), 256, 0, st>>>(bottom_diff, n_in);
    int bins = pooled_height * pooled_width;
    if (num_rois > 0 && bins > 0) {
        int out_ch = pool_channel ? 1 : channels;
        if (out_ch % 4 == 0 && aligned16(top_diff) && aligned16(argmax)) {
            size_t total = (size_t)num_rois * bins * (out_ch / 4);
            k_roi_pool_bwd<4><<<grid_for(total, 256), 256, 0, st>>>(top_diff, argmax, rois, batch, num_rois, channel_rois,
                                                                    height, width, channels, out_ch, pooled_height,
                                                                    pooled_width, spatial_scale, bottom_diff);
        } else {
            size_t total = (size_t)num_rois * bins * out_ch;
            k_roi_pool_bwd<1><<<grid_for(total, 256), 256, 0, st>>>(top_diff, argmax, rois, batch, num_rois, channel_rois,
                                                                    height, width, channels, out_ch, pooled_height,
                                                                    pooled_width, spatial_scale, bottom_diff);
        }
    }
    return check_launch("roi_pool_bwd");
}

extern "C" int pcnn_hard_label_fwd(const float* prob, const int32_t* gt, int B, int H, int W, int C, float threshold,
                                   float* top, void* stream)
{
    PCNN_REQUIRE(prob && gt && top, "hard_label: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 1, "hard_label: bad shape");
    PCNN_REQUIRE(aligned16(top), "hard_label: output must be 16-byte aligned");
    size_t npix = (size_t)B * H * W;
    k_hard_label<<<grid_for(npix * C / 4 + 1, 256), 256, 0, (cudaStream_t)stream>>>(prob, gt, npix, C, threshold, top);
    return check_launch("hard_label_fwd");
}

extern "C" int pcnn_hard_label_bwd(int B, int H, int W, int C, float* grad_prob, float* grad_gt, void* stream)
{
    PCNN_REQUIRE(grad_prob && grad_gt, "hard_label_grad: NULL tensor pointer");
    size_t npix = (size_t)B * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    k_fill_zero<<<grid_for(npix * C / 4 + 1, 256), 256, 0, st>>>(grad_prob, npix * C);
    k_fill_zero<<<grid_for(npix / 4 + 1, 256), 256, 0, st>>>(grad_gt, npix);
    return check_launch("hard_label_bwd");
}

static int launch_gather(const float* vox, const float* depth, const float* meta, int B, int H, int W, int Cf,
                         int num_meta, int G, float* out, cudaStream_t st)
{
    if ((size_t)H * W * Cf >= 0x7fffffffULL || B > 65535) { set_error("project: image too large for 32-bit indexing"); return PCNN_E_INVALID; }
    if (Cf % 4 == 0 && aligned16(vox) && aligned16(out)) {
        size_t total = (size_t)H * W * (Cf / 4);
        k_pixel_gather<4><<<dim3(grid_for(total, 256, 8), B), 256, 0, st>>>(vox, depth, meta, B, H, W, Cf, num_meta, G, out);
    } else {
        size_t total = (size_t)H * W * Cf;
        k_pixel_gather<1><<<dim3(grid_for(total, 256, 8), B), 256, 0, st>>>(vox, depth, meta, B, H, W, Cf, num_meta, G, out);
    }
    return check_launch("pixel gather");
}

static int launch_average(const float* src, const float* depth, const float* meta, const float* fallback, int B, int H,
                          int W, int nch, int num_meta, int G, int ks, float thr, float* dst, float* flag, cudaStream_t st)
{
    bool v4 = nch % 4 == 0 && aligned16(src) && aligned16(dst) && (!fallback || aligned16(fallback)) &&
              (!flag || aligned16(flag));
    if ((size_t)G * G * G * nch >= 0x7fffffffULL || B > 65535) { set_error("backproject: grid too large for 32-bit indexing"); return PCNN_E_INVALID; }
    if (v4 && nch % 16 == 0) {
        size_t total = (size_t)G * G * G * (nch / 16);
        k_voxel_average_wide<16, false><<<dim3(grid_for(total, 256, 8), B), 256, 0, st>>>(src, depth, meta, fallback, H, W, nch, num_meta,
                                                                                         G, ks, thr, dst, flag);
        return check_launch("voxel average (16 channels / thread)");
    }
    if (!v4 && nch <= 32) {
        size_t total = (size_t)G * G * G;
        k_voxel_average_wide<32, true><<<dim3(grid_for(total, 256, 8), B), 256, 0, st>>>(src, depth, meta, fallback, H, W, nch, num_meta,
                                                                                        G, ks, thr, dst, flag);
        return check_launch("voxel average (whole voxel / thread)");
    }
    if (v4) {
        size_t total = (size_t)G * G * G * (nch / 4);
        k_voxel_average<4><<<dim3(grid_for(total, 256, 8), B), 256, 0, st>>>(src, depth, meta, fallback, B, H, W, nch, num_meta, G,
                                                                             ks, thr, dst, flag);
    } else {
        size_t total = (size_t)G * G * G * nch;
        k_voxel_average<1><<<dim3(grid_for(total, 256, 8), B), 256, 0, st>>>(src, depth, meta, fallback, B, H, W, nch, num_meta, G,
                                                                             ks, thr, dst, flag);
    }
    return check_launch("voxel average");
}

extern "C" int pcnn_backproject_fwd(const float* data, const float* label, const float* depth, const float* meta,
                                    const float* label_3d, int B, int H, int W, int Cf, int C, int num_meta,
                                    int grid_size, int kernel_size, float threshold, float* top_data,
                                    float* top_label, float* top_flag, void* stream)
{
    PCNN_REQUIRE(grid_size >= 0, "Need grid_size >= 0, got %d", grid_size);        // backprojecting_op.cc:303-305
    PCNN_REQUIRE(kernel_size >= 0, "Need kernel_size >= 0, got %d", kernel_size);  // :310-312
    PCNN_REQUIRE(threshold >= 0, "Need threshold >= 0, got %f", threshold);        // :317-319
    PCNN_REQUIRE(num_meta >= 48, "backproject: meta_data needs 48 floats (got %d)", num_meta);
    PCNN_REQUIRE(data && label && depth && meta && label_3d && top_data && top_label && top_flag,
                 "backproject: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && Cf >= 1 && C >= 1, "backproject: bad shape");
    if (grid_size == 0) return PCNN_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        const size_t G3 = (size_t)grid_size * grid_size * grid_size;
        static const bool fused_on = getenv("PCNN_BACKPROJECT_FUSED") == nullptr || atoi(getenv("PCNN_BACKPROJECT_FUSED")) != 0;
        if (fused_on && Cf % 4 == 0 && aligned16(data) && aligned16(top_data) && aligned16(top_flag) && B <= 65535 &&
            G3 * (size_t)(Cf > C ? Cf : C) < 0x7fffffffULL) {
            dim3 grid((unsigned)((G3 + kBpVox - 1) / kBpVox), B);
            k_backproject_fused<<<grid, 256, 0, st>>>(data, label, depth, meta, label_3d, H, W, Cf, C, num_meta, grid_size, kernel_size,
                                                      threshold, top_data, top_label, top_flag);
            return check_launch("backproject (fused)");
        }
    }
    int rc = launch_average(data, depth, meta, nullptr, B, H, W, Cf, num_meta, grid_size, kernel_size, threshold, top_data,
                            top_flag, st);
    if (rc) return rc;
    return launch_average(label, depth, meta, label_3d, B, H, W, C, num_meta, grid_size, kernel_size, threshold, top_label,
                          nullptr, st);
}

extern "C" int pcnn_backproject_bwd(const float* top_diff, const float* depth, const float* meta, int B, int H, int W,
                                    int Cf, int num_meta, int grid_size, float* bottom_diff, void* stream)
{
    PCNN_REQUIRE(top_diff && depth && meta && bottom_diff, "backproject_grad: NULL tensor pointer");
    PCNN_REQUIRE(num_meta >= 48 && grid_size >= 1, "backproject_grad: bad meta/grid");
    return launch_gather(top_diff, depth, meta, B, H, W, Cf, num_meta, grid_size, bottom_diff, (cudaStream_t)stream);
}

extern "C" int pcnn_project_fwd(const float* data, const float* depth, const float* meta, int B, int H, int W, int Cf,
                                int num_meta, int grid_size, float* top, void* stream)
{
    PCNN_REQUIRE(data && depth && meta && top, "project: NULL tensor pointer");
    PCNN_REQUIRE(num_meta >= 48 && grid_size >= 1, "project: bad meta/grid");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && Cf >= 1, "project: bad shape");
    return launch_gather(data, depth, meta, B, H, W, Cf, num_meta, grid_size, top, (cudaStream_t)stream);
}

extern "C" int pcnn_project_bwd(const float* top_diff, const float* depth, const float* meta, int B, int H, int W,
                                int Cf, int num_meta, int grid_size, int kernel_size, float threshold,
                                float* bottom_diff, void* stream)
{
    PCNN_REQUIRE(top_diff && depth && meta && bottom_diff, "project_grad: NULL tensor pointer");
    PCNN_REQUIRE(kernel_size >= 0, "Need kernel_size >= 0, got %d", kernel_size);  // projecting_op.cc:226-228
    PCNN_REQUIRE(threshold >= 0, "Need threshold >= 0, got %f", threshold);
    PCNN_REQUIRE(num_meta >= 48 && grid_size >= 1, "project_grad: bad meta/grid");
    return launch_average(top_diff, depth, meta, nullptr, B, H, W, Cf, num_meta, grid_size, kernel_size, threshold,
                          bottom_diff, nullptr, (cudaStream_t)stream);
}

// RoiPool forward on bf16 NHWC features (channels % 8 == 0), fp32 top + int32 argmax
extern "C" int pcnn_roi_pool_fwd_bf16(const void* bottom_bf16, const float* rois, int num_rois, int channel_rois, int batch,
                                      int height, int width, int channels, int pooled_height, int pooled_width,
                                      float spatial_scale, float* top, int32_t* argmax, void* stream)
{
    PCNN_REQUIRE(bottom_bf16 && rois && top && argmax, "roi_pool_bf16: NULL tensor pointer");
    PCNN_REQUIRE(channel_rois >= 6 && channels % 8 == 0, "roi_pool_bf16: needs >= 6 roi columns and channels %% 8 == 0");
    if (num_rois == 0 || pooled_height == 0 || pooled_width == 0) return PCNN_OK;
    size_t total = (size_t)num_rois * pooled_height * pooled_width * (channels / 8);
    if (channels % 32 == 0 && height * width < 0xffff &&
        (long long)num_rois * pooled_height * pooled_width * (channels / 32) * 32 < 0x7fffffffLL) {
        size_t threads = (size_t)num_rois * pooled_height * pooled_width * (channels / 32) * 32;
        k_roi_pool_fwd_bf16_s4<<<grid_for(threads, 256), 256, 0, (cudaStream_t)stream>>>(
            (const __nv_bfloat16*)bottom_bf16, rois, num_rois, channel_rois, batch, height, width, channels, pooled_height,
            pooled_width, spatial_scale, top, argmax);
        return check_launch("roi_pool_fwd_bf16_s4");
    }
    k_roi_pool_fwd_bf16<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)bottom_bf16, rois, num_rois, channel_rois, batch, height, width, channels, pooled_height,
        pooled_width, spatial_scale, top, argmax);
    return check_launch("roi_pool_fwd_bf16");
}
