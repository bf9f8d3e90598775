// heads.cu — the FCN heads of vgg16_convs after the 1x1 convolutions on conv4_3 / conv5_3:
// semantic-label head and vertex head (lib/networks/vgg16_convs.py:128-163).
//
// The reference runs, at FULL resolution, two dense conv2d_transpose ops whose filters are fixed
// diagonal bilinear kernels (make_deconv_filter, lib/networks/network.py:141-157, 207-222) followed by
// 1x1 convolutions (`score` 64->C with ReLU, `vertex_pred` 128->3C): 50 GFLOP/frame of multiplications
// by zero plus 6 GFLOP of 1x1 work on 307 200 pixels.  Both stages are linear and act on different
// axes (bilinear: per channel over space; 1x1: per pixel over channels), so they commute:
//
//      conv1x1(up8(x)) + b  ==  up8(conv1x1_nobias(x)) + b
//
// (the bias must stay outside: near the image border the transposed convolution's weights do not sum
// to one).  Hence:
//   k_lowres_heads  at 1/8 resolution: add_score = score_conv4 + up2(score_conv5) (both heads), then
//                   the two 1x1 matrices -> [B,h,w, C + 3C] fp32
//   k_up8_heads     per output pixel: bilinear x8 (exact conv2d_transpose weights), + bias, ReLU /
//                   softmax / arg-max for the label head, + bias for the vertex head; one streaming
//                   pass that writes label_2d (int32), vertex_pred (fp32) and optionally the
//                   normalised probabilities.
#include <cuda_bf16.h>
#include <float.h>

#include <algorithm>

#include "common.cuh"
#include "heads_common.cuh"

namespace pcnn {

// ---------------------------------------------------------------------------------------------
// k_lowres_heads: one warp per group of 8 consecutive low-resolution pixels.
//   phase 1  lane (q = lane & 7, g = lane >> 3) builds pixel q's two "add" vectors (conv4 branch + 4x4/2
//            transposed convolution of the conv5 branch; 8-byte bf16x4 reads) into the warp's shared-memory
//            slot, channel-major: sx[ch][8 pixels].
//   phase 2  register-tiled matrix products: every lane owns one output column for all 8 pixels, so one k step
//            costs 1 weight word + 2 broadcast float4 of activations for 8 FMAs.  The 4C outputs are covered in
//            three passes of <= 32 columns: vertex 0..31, vertex 32..63 (K = Cv), then the C score columns
//            (K = Cs) next to the remaining vertex columns, each of those split over Cv/Cs lanes of Cs rows and
//            summed by shuffle, so no lane idles behind a longer loop.
// Requires Cs % 4 == 0, Cv % Cs == 0 (64 / 128 in the network).
// kVertex = false: the segmentation network's score-only head tensor [B,h,w,C] (no vertex head, vgg16_convs.py:128-149 with the
// vertex block skipped): v4 / v5 / Wv are not read, phase 1 stages the Cs score channels and phase 2 is the score-column tail pass.
// ---------------------------------------------------------------------------------------------
constexpr int kLrWarps = 8;
constexpr int kLrPix = 8;

template <bool kVertex>
__global__ void __launch_bounds__(256)
k_lowres_heads(const __nv_bfloat16* __restrict__ s4 /*[B,h,w,Cs]*/, const __nv_bfloat16* __restrict__ s5 /*[B,h/2,w/2,Cs]*/,
               const __nv_bfloat16* __restrict__ v4 /*[B,h,w,Cv]*/, const __nv_bfloat16* __restrict__ v5,
               const float* __restrict__ Ws /*[Cs][C]*/, const float* __restrict__ Wv /*[Cv][3C]*/, int B, int h, int w,
               int Cs, int Cv, int C, float* __restrict__ out /*[B,h,w,4C], score-only [B,h,w,C]*/)
{
    extern __shared__ __align__(16) float sm[];
    // folded mode (Wv == NULL): the vertex_pred matrix was multiplied into the two vertex 1x1 convolutions on the host
    // (both are linear, no ReLU between them), so v4 / v5 already hold the 3C vertex channels (row stride Cv) and the
    // vertex outputs are just v4 + up2(v5)
    const bool folded = kVertex && Wv == nullptr;
    const int Ct = folded || !kVertex ? Cs : Cs + Cv;   // channels staged in shared memory
    const int No = kVertex ? 4 * C : C;                 // outputs per pixel
    const int C3 = folded || !kVertex ? 0 : 3 * C;      // vertex columns of the matrix phase
    float* sx_all = sm;                               // [kLrWarps][Ct][8]   (16-byte aligned rows)
    float* sW = sm + kLrWarps * Ct * kLrPix;          // [Cs*C + Cv*3C]
    for (int i = threadIdx.x; i < Cs * C; i += blockDim.x) sW[i] = Ws[i];
    if (kVertex && !folded)
        for (int i = threadIdx.x; i < Cv * C3; i += blockDim.x) sW[Cs * C + i] = Wv[i];
    __syncthreads();
    const float* sWv = sW + Cs * C;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* sx = sx_all + warp * Ct * kLrPix;
    const int npix = B * h * w;
    const int h5 = h / 2, w5 = w / 2;
    const int ngroups = (npix + kLrPix - 1) / kLrPix;
    const int q = lane & 7, g = lane >> 3;
    const int nquads = Ct / 4;
    // column map: n_full passes of 32 vertex columns (K = Cv); then "tail" passes whose lane jobs are the C score
    // columns (K = Cs) followed, from a split-aligned start, by split = Cv / Cs partial lanes per left-over vertex column
    const int split = kVertex ? Cv / Cs : 1;
    const int n_full = C3 / 32, v_left = C3 - 32 * n_full;
    const int tail_start = (C + split - 1) / split * split;
    const int n_pass = n_full + (tail_start + v_left * split + 31) / 32;
    for (int grp = blockIdx.x * kLrWarps + warp; grp < ngroups; grp += gridDim.x * kLrWarps) {
        // ---- phase 1: add = conv4 branch + up2(conv5 branch): conv2d_transpose 4x4 / stride 2, SAME (pad 1)
        {
            const int p = grp * kLrPix + q;
            const bool live = p < npix;
            const int pc = live ? p : npix - 1;
            const int x = pc % w, y = (pc / w) % h, n = pc / (w * h);
            // out[o] += in[i] * W[o - 2 i + 1], 0 <= o - 2i + 1 <= 3: two source rows / columns
            const int iy0 = ((y + 1) >> 1) - 1, ix0 = ((x + 1) >> 1) - 1;
            float wgt[4];
            int off5[4];
#pragma unroll
            for (int d = 0; d < 4; d++) {
                const int iy = iy0 + (d >> 1), ix = ix0 + (d & 1);
                const int ky = y - 2 * iy + 1, kx = x - 2 * ix + 1;
                const bool ok = iy >= 0 && iy < h5 && ix >= 0 && ix < w5;
                wgt[d] = ok ? deconv_w(ky, 4) * deconv_w(kx, 4) : 0.f;
                off5[d] = (n * h5 + min(max(iy, 0), h5 - 1)) * w5 + min(max(ix, 0), w5 - 1);
            }
            for (int qd = g; qd < nquads; qd += 4) {
                const int ch = 4 * qd;
                const bool vert = ch >= Cs;
                const int cc = vert ? ch - Cs : ch, Cn = vert ? Cv : Cs;
                const __nv_bfloat16* a = vert ? v4 : s4;
                const __nv_bfloat16* b5 = vert ? v5 : s5;
                const uint2 ua = __ldg(reinterpret_cast<const uint2*>(a + (size_t)pc * Cn + cc));
                float acc[4];
                {
                    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&ua.x), hi = *reinterpret_cast<const __nv_bfloat162*>(&ua.y);
                    acc[0] = __low2float(lo); acc[1] = __high2float(lo); acc[2] = __low2float(hi); acc[3] = __high2float(hi);
                }
                float up[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int d = 0; d < 4; d++) {
                    const uint2 ub = __ldg(reinterpret_cast<const uint2*>(b5 + (size_t)off5[d] * Cn + cc));
                    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&ub.x), hi = *reinterpret_cast<const __nv_bfloat162*>(&ub.y);
                    if (d == 0) {
                        up[0] = wgt[0] * __low2float(lo); up[1] = wgt[0] * __high2float(lo);
                        up[2] = wgt[0] * __low2float(hi); up[3] = wgt[0] * __high2float(hi);
                    } else {
                        up[0] = fmaf(wgt[d], __low2float(lo), up[0]); up[1] = fmaf(wgt[d], __high2float(lo), up[1]);
                        up[2] = fmaf(wgt[d], __low2float(hi), up[2]); up[3] = fmaf(wgt[d], __high2float(hi), up[3]);
                    }
                }
#pragma unroll
                for (int i = 0; i < 4; i++) sx[(ch + i) * kLrPix + q] = live ? acc[i] + up[i] : 0.f;
            }
            if (folded && live) {
                // vertex outputs straight to HBM: channels [4 qd, 4 qd + 4) of the 3C (tensor rows are zero padded to Cv)
                float* op = out + (size_t)p * No + C;
                const int nvq = (3 * C + 3) / 4;
                for (int qd = g; qd < nvq; qd += 4) {
                    const int cc = 4 * qd;
                    const uint2 ua = __ldg(reinterpret_cast<const uint2*>(v4 + (size_t)pc * Cv + cc));
                    const __nv_bfloat162 alo = *reinterpret_cast<const __nv_bfloat162*>(&ua.x), ahi = *reinterpret_cast<const __nv_bfloat162*>(&ua.y);
                    float r[4] = {__low2float(alo), __high2float(alo), __low2float(ahi), __high2float(ahi)};
                    float up[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int d = 0; d < 4; d++) {
                        const uint2 ub = __ldg(reinterpret_cast<const uint2*>(v5 + (size_t)off5[d] * Cv + cc));
                        const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&ub.x), hi = *reinterpret_cast<const __nv_bfloat162*>(&ub.y);
                        if (d == 0) {
                            up[0] = wgt[0] * __low2float(lo); up[1] = wgt[0] * __high2float(lo);
                            up[2] = wgt[0] * __low2float(hi); up[3] = wgt[0] * __high2float(hi);
                        } else {
                            up[0] = fmaf(wgt[d], __low2float(lo), up[0]); up[1] = fmaf(wgt[d], __high2float(lo), up[1]);
                            up[2] = fmaf(wgt[d], __low2float(hi), up[2]); up[3] = fmaf(wgt[d], __high2float(hi), up[3]);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        if (cc + i < 3 * C) op[cc + i] = r[i] + up[i];
                }
            }
        }
        __syncwarp();
        // ---- phase 2
        const int p0 = grp * kLrPix;
        const int nlive = min(kLrPix, npix - p0);
        float* obase = out + (size_t)p0 * No;
#pragma unroll 1
        for (int pass = 0; pass < n_pass; pass++) {
            // column / K-range of this lane in this pass
            const float* wp;      // weight of (k = 0) for this lane's column, stride ld
            const float* xp;      // activations of (k = 0)
            int ld, kn, col;      // col = output index within the 4C outputs, or -1 (idle)
            bool partial = false; // tail vertex lanes hold a partial sum
            if (pass < n_full) {
                const int vc = 32 * pass + lane;
                col = C + vc; wp = sWv + vc; ld = C3; kn = Cv; xp = sx + Cs * kLrPix;
            } else {
                const int job = 32 * (pass - n_full) + lane;
                kn = Cs;
                if (job < C) {
                    col = job; wp = sW + job; ld = C; xp = sx;
                } else {
                    const int j = job - tail_start;
                    const bool ok = j >= 0 && j < v_left * split;
                    const int vc = ok ? 32 * n_full + j / split : 0, part = ok ? j % split : 0;
                    col = ok ? C + vc : -1; partial = ok;
                    wp = ok ? sWv + (size_t)(part * Cs) * C3 + vc : sW; ld = ok ? C3 : 0;   // idle lanes re-read one valid word
                    xp = ok ? sx + (Cs + part * Cs) * kLrPix : sx;
                }
            }
            float acc[kLrPix];
#pragma unroll
            for (int i = 0; i < kLrPix; i++) acc[i] = 0.f;
#pragma unroll 4
            for (int k = 0; k < kn; k++) {
                const float wk = wp[k * ld];
                const float4 x0 = *reinterpret_cast<const float4*>(xp + k * kLrPix);
                const float4 x1 = *reinterpret_cast<const float4*>(xp + k * kLrPix + 4);
                acc[0] = fmaf(x0.x, wk, acc[0]); acc[1] = fmaf(x0.y, wk, acc[1]);
                acc[2] = fmaf(x0.z, wk, acc[2]); acc[3] = fmaf(x0.w, wk, acc[3]);
                acc[4] = fmaf(x1.x, wk, acc[4]); acc[5] = fmaf(x1.y, wk, acc[5]);
                acc[6] = fmaf(x1.z, wk, acc[6]); acc[7] = fmaf(x1.w, wk, acc[7]);
            }
            if (pass >= n_full && split > 1) {
                // sum the `split` adjacent partial lanes of a left-over vertex column (split is a power of two)
                for (int d = 1; d < split; d <<= 1) {
#pragma unroll
                    for (int i = 0; i < kLrPix; i++) {
                        const float o = __shfl_down_sync(0xffffffffu, acc[i], d);
                        if (partial) acc[i] += o;
                    }
                }
                if (partial && ((32 * (pass - n_full) + lane - tail_start) % split) != 0) col = -1;
            }
            if (col >= 0) {
#pragma unroll
                for (int i = 0; i < kLrPix; i++)
                    if (i < nlive) obase[(size_t)i * No + col] = acc[i];
            }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// k_up8_heads: one CTA per (output row, image, segment of low-resolution cells).  The two contributing
// low-resolution rows are combined vertically into shared memory once; every output value is then a 2-tap horizontal
// blend with compile-time weights.  Class scores of the segment are kept in shared memory for the per-pixel arg-max /
// softmax.  CT = compile-time class count (0 = run-time): with CT fixed every store address of a thread is
// `base + immediate`, which is what takes this kernel from instruction-bound to store-bound (ncu: 1.29 G warp
// instructions, 24 % of them IMAD address math, before the change).
// Thread roles: threads [0, nv) own one vertex channel pair of one cell phase (consecutive lanes = consecutive channel
// pairs -> contiguous 8-byte stores), threads [nv, nv + ns) own one score channel pair.
// CPT = channels per thread.  2: C even, the roles above.  1: C odd, where a pixel's score row, its vertex row and the vertex
// part of a low-resolution row are not 8-byte aligned: a role owns ONE channel (4-byte loads and stores, consecutive lanes still
// on consecutive channels), so a cell phase takes 4C roles; at C >= 65 that exceeds the CTA and a thread loops over the roles
// with stride 256.
// kVertex = false: lr is the segmentation network's score-only head tensor [B,h,w,C] (row stride C instead of 4C); vertex is NULL.
// ---------------------------------------------------------------------------------------------
template <int CT, int CPT, bool kVertex>
__global__ void __launch_bounds__(256)
k_up8_heads(const float* __restrict__ lr /*[B,h,w,4C] or [B,h,w,C]*/, const float* __restrict__ bias_s /*[C]*/,
            const float* __restrict__ bias_v /*[3C]*/, int h, int w, int C_rt, int seg_cells, int* __restrict__ label /*[B,8h,8w]*/,
            float* __restrict__ vertex /*[B,8h,8w,3C]*/, float* __restrict__ prob /*[B,8h,8w,C] or null*/,
            float* __restrict__ score_out /*[B,8h,8w,C] or null*/)
{
    // CPT = 2, C even: every channel pair is one 8-byte vector (vertex rows are 3C floats = 8-byte aligned).
    extern __shared__ float smem_f[];
    const int C = CT ? CT : C_rt;
    const int No = (kVertex ? 4 : 1) * C, W = 8 * w, H = 8 * h, N2 = No / 2, C2 = C / 2, V2 = 3 * C2;
    const int c_lo = blockIdx.z * seg_cells, c_hi = min(c_lo + seg_cells, w);   // cells [c_lo, c_hi)
    const int s_lo = max(c_lo - 1, 0), s_hi = min(c_hi + 1, w);                 // source cells incl. halo
    float2* rowi = reinterpret_cast<float2*>(smem_f) - (size_t)s_lo * N2;       // [s_lo, s_hi) x N2, indexed by absolute cell
    float* sc = smem_f + (size_t)(seg_cells + 2) * No - (size_t)8 * c_lo * C;   // [8 seg_cells][C], indexed by absolute x
    float* stat = smem_f + (size_t)(seg_cells + 2) * No + (size_t)8 * seg_cells * C;   // [8 seg_cells][2]: softmax max / sum of a pixel
    const int y = blockIdx.x, n = blockIdx.y, t = threadIdx.x;
    // conv2d_transpose 16x16 / stride 8, SAME (pad 4): out[o] = sum_i in[i] * W[o - 8i + 4]
    const int my = y >> 3, ty = y & 7;
    const int iy0 = ty < 4 ? my - 1 : my, iy1 = iy0 + 1;
    const float wy0 = (iy0 >= 0 && iy0 < h) ? deconv_w(y - 8 * iy0 + 4, 16) : 0.f;
    const float wy1 = (iy1 >= 0 && iy1 < h) ? deconv_w(y - 8 * iy1 + 4, 16) : 0.f;
    const float2* r0 = reinterpret_cast<const float2*>(lr + ((size_t)n * h + min(max(iy0, 0), h - 1)) * w * No);
    const float2* r1 = reinterpret_cast<const float2*>(lr + ((size_t)n * h + min(max(iy1, 0), h - 1)) * w * No);
    if constexpr (CPT == 1) {
        float* rows = smem_f - (size_t)s_lo * No;                                   // [s_lo, s_hi) x No scalars
        const float* q0 = reinterpret_cast<const float*>(r0);
        const float* q1 = reinterpret_cast<const float*>(r1);
        if (vertex) {
            for (int i = s_lo * No + t; i < s_hi * No; i += 256) rows[i] = up8_vblend(wy0, __ldg(q0 + i), wy1, __ldg(q1 + i));
        } else {
            for (int j = t; j < (s_hi - s_lo) * C; j += 256) {
                const int i = (s_lo + j / C) * No + j % C;
                rows[i] = up8_vblend(wy0, __ldg(q0 + i), wy1, __ldg(q1 + i));
            }
        }
    } else if (vertex) {
        for (int i = s_lo * N2 + t; i < s_hi * N2; i += 256) {
            const float2 a = __ldg(r0 + i), b = __ldg(r1 + i);
            rowi[i] = make_float2(up8_vblend(wy0, a.x, wy1, b.x), up8_vblend(wy0, a.y, wy1, b.y));
        }
    } else {   // label-only mode (the pipeline's Hough samples its vertex values from `lowres` itself): score channels only
        for (int j = t; j < (s_hi - s_lo) * C2; j += 256) {
            const int i = (s_lo + j / C2) * N2 + j % C2;
            const float2 a = __ldg(r0 + i), b = __ldg(r1 + i);
            rowi[i] = make_float2(up8_vblend(wy0, a.x, wy1, b.x), up8_vblend(wy0, a.y, wy1, b.y));
        }
    }
    __syncthreads();
    const size_t rowbase = ((size_t)n * H + y) * W;
    const float2 zero = make_float2(0.f, 0.f);
    // x = 8 mx + tx: sources (mx-1, mx) with taps (tx+12, tx+4) for tx < 4, (mx, mx+1) with (tx+4, tx-4) otherwise
#define PCNN_UP8_BLEND(tx, v0, v1)                                                                             \
    const float wa = deconv_w(tx < 4 ? tx + 12 : tx + 4, 16), wb = deconv_w(tx < 4 ? tx + 4 : tx - 4, 16);     \
    const float2 a = tx < 4 ? vl : vc, b = tx < 4 ? vc : vr;                                                   \
    float v0 = up8_hblend(wa, a.x, wb, b.x, bb.x);                                                             \
    float v1 = up8_hblend(wa, a.y, wb, b.y, bb.y);
    if constexpr (CPT == 1) {
        // one channel per role: vertex roles [0, gv 3C), score roles [gv 3C, gv 4C); label-only mode: score roles only
        const float* rows = smem_f - (size_t)s_lo * No;
        const int gv = vertex ? max(256 / No, 1) : min(256 / C, seg_cells);
        const int nv = vertex ? gv * 3 * C : 0;
        for (int u = t; u < nv + gv * C; u += 256) {
            const bool vrole = u < nv;
            const int uc = vrole ? u : u - nv, Cr = vrole ? 3 * C : C;
            const int g = uc / Cr, c = uc - g * Cr;
            const float bb = vrole ? bias_v[c] : bias_s[c];
            const float* src = rows + (vrole ? C : 0) + c;
            float* op = vrole ? vertex + (rowbase + 8 * (size_t)(c_lo + g)) * 3 * C + c : sc + 8 * (c_lo + g) * C + c;
            float* gp = !vrole && score_out ? score_out + (rowbase + 8 * (size_t)(c_lo + g)) * C + c : nullptr;
            for (int mx = c_lo + g; mx < c_hi; mx += gv, op += gv * 8 * Cr) {
                const float vl = mx > 0 ? src[(mx - 1) * No] : 0.f;
                const float vc = src[mx * No];
                const float vr = mx + 1 < w ? src[(mx + 1) * No] : 0.f;
#pragma unroll
                for (int tx = 0; tx < 8; tx++) {
                    const float wa = deconv_w(tx < 4 ? tx + 12 : tx + 4, 16), wb = deconv_w(tx < 4 ? tx + 4 : tx - 4, 16);
                    const float v = up8_hblend(wa, tx < 4 ? vl : vc, wb, tx < 4 ? vc : vr, bb);
                    if (vrole) {
                        __stcs(op + tx * 3 * C, v);
                    } else {
                        op[tx * C] = fmaxf(v, 0.f);                       // `score` has a ReLU
                        if (gp) gp[tx * C] = fmaxf(v, 0.f);
                    }
                }
                if (gp) gp += gv * 8 * C;
            }
        }
    } else {
        // cell phases; vertex threads [0, gv*V2), score threads [gv*V2, gv*N2); label-only mode: all threads on scores
        const int gv = vertex ? 256 / N2 : min(256 / C2, seg_cells);
        const int nv = vertex ? gv * V2 : 0;
        if (t < nv) {
            const int g = t / V2, c2 = t - g * V2;                   // vertex channel pair c2 (channels C + 2 c2, +1 of a lowres cell)
            const float2 bb = make_float2(bias_v[2 * c2], bias_v[2 * c2 + 1]);
            const float2* src = rowi + C2 + c2;
            float* vp = vertex + (rowbase + 8 * (size_t)(c_lo + g)) * 3 * C + 2 * c2;
            const int vstep = gv * 8 * 3 * C;
            for (int mx = c_lo + g; mx < c_hi; mx += gv, vp += vstep) {
                const float2 vl = mx > 0 ? src[(mx - 1) * N2] : zero;
                const float2 vc = src[mx * N2];
                const float2 vr = mx + 1 < w ? src[(mx + 1) * N2] : zero;
#pragma unroll
                for (int tx = 0; tx < 8; tx++) {
                    PCNN_UP8_BLEND(tx, v0, v1)
                    __stcs(reinterpret_cast<float2*>(vp + tx * 3 * C), make_float2(v0, v1));
                }
            }
        } else if (t < nv + gv * C2) {
            const int u = t - nv;
            const int g = u / C2, c2 = u - g * C2;                   // score channel pair
            const float2 bb = make_float2(bias_s[2 * c2], bias_s[2 * c2 + 1]);
            const float2* src = rowi + c2;
            float* sp = sc + 8 * (c_lo + g) * C + 2 * c2;
            float* gp = score_out ? score_out + (rowbase + 8 * (size_t)(c_lo + g)) * C + 2 * c2 : nullptr;
            for (int mx = c_lo + g; mx < c_hi; mx += gv, sp += gv * 8 * C) {
                const float2 vl = mx > 0 ? src[(mx - 1) * N2] : zero;
                const float2 vc = src[mx * N2];
                const float2 vr = mx + 1 < w ? src[(mx + 1) * N2] : zero;
#pragma unroll
                for (int tx = 0; tx < 8; tx++) {
                    PCNN_UP8_BLEND(tx, v0, v1)
                    v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);        // `score` has a ReLU (vgg16_convs.py:141, network.py:160)
                    *reinterpret_cast<float2*>(sp + tx * C) = make_float2(v0, v1);
                    if (gp) *reinterpret_cast<float2*>(gp + tx * C) = make_float2(v0, v1);
                }
                if (gp) gp += gv * 8 * C;
            }
        }
    }
#undef PCNN_UP8_BLEND
    __syncthreads();
    // arg-max over classes, lowest index wins ties (tf.argmax); softmax for prob_normalized (network.py:474-488)
    for (int x = 8 * c_lo + t; x < 8 * c_hi; x += 256) {
        float best;
        int bi = 0;
        if constexpr (CPT == 1) {
            const float* s1 = sc + x * C;
            best = s1[0];
            for (int c = 1; c < C; c++)
                if (s1[c] > best) { best = s1[c]; bi = c; }
        } else {
            const float2* s2 = reinterpret_cast<const float2*>(sc + x * C);
            best = s2[0].x;
            if (s2[0].y > best) { best = s2[0].y; bi = 1; }
#pragma unroll
            for (int c = 1; c < (CT ? CT / 2 : 1); c++) {
                const float2 v = s2[c];
                if (v.x > best) { best = v.x; bi = 2 * c; }
                if (v.y > best) { best = v.y; bi = 2 * c + 1; }
            }
            if (!CT)
                for (int c = 1; c < C2; c++) {
                    const float2 v = s2[c];
                    if (v.x > best) { best = v.x; bi = 2 * c; }
                    if (v.y > best) { best = v.y; bi = 2 * c + 1; }
                }
        }
        label[rowbase + x] = bi;
        if (prob) {
            // softmax statistics of the pixel; the normalised row is written by the cooperative pass below
            const float* s = sc + x * C;
            float sum = 0.f;
            for (int c = 0; c < C; c++) sum += expf(s[c] - best);
            stat[2 * (x - 8 * c_lo)] = best;
            stat[2 * (x - 8 * c_lo) + 1] = sum;
        }
    }
    if (prob) {
        // prob_normalized = exp(s - max) / sum (network.py:474-488), thread = (pixel, class) in memory order: the segment's
        // 8 (c_hi - c_lo) * C floats are one contiguous run of the output row -> coalesced stores (thread = pixel wrote C floats
        // 88 B apart: 22 store instructions of 32 scattered sectors each)
        __syncthreads();
        const int nel = 8 * (c_hi - c_lo) * C;
        const float* s = sc + (size_t)8 * c_lo * C;
        float* pr = prob + (rowbase + 8 * (size_t)c_lo) * C;
        for (int i = t; i < nel; i += 256) {
            const int xl = i / C;
            pr[i] = expf(s[i] - stat[2 * xl]) / stat[2 * xl + 1];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// k_up8_label: label-only form of k_up8_heads for the pipeline (Hough samples its vertex values from `lowres`): one CTA per
// (low-resolution row, image) produces the EIGHT output rows that row owns.  The three contributing low-resolution rows'
// score channels are staged once (k_up8_heads re-stages two rows for every output row); per output row, thread =
// (cell, class pair) blends vertically in registers, emits the cell's 8 pixels into a shared score row, and thread =
// pixel takes the arg-max (lowest index on ties).  Same operation sequence as k_up8_heads (heads_common.cuh): identical
// labels.  CT = compile-time class count (even), CPT = channels per thread as in k_up8_heads: at CPT = 1 (C odd) the staged rows
// are [3][w][C] scalars and a thread blends (cell, class).  kVertex as in k_up8_heads (row stride 4C or C).
// ---------------------------------------------------------------------------------------------
// 512 threads: the kernel is latency-bound (shared-memory chains between two barriers per output row); with 77 KB of shared
// memory per CTA only two CTAs fit an SM, so the warps have to come from the CTA itself
constexpr int kLabelThreads = 512;

template <int CT, int CPT, bool kVertex>
__global__ void __launch_bounds__(kLabelThreads)
k_up8_label(const float* __restrict__ lr /*[B,h,w,4C] or [B,h,w,C]*/, const float* __restrict__ bias_s /*[C]*/, int h, int w, int C_rt,
            int* __restrict__ label /*[B,8h,8w]*/)
{
    extern __shared__ float smem_f[];
    const int C = CT ? CT : C_rt;
    const int No = (kVertex ? 4 : 1) * C, C2 = C / 2, W = 8 * w;
    float2* rows = reinterpret_cast<float2*>(smem_f);              // [3][w][C2]: low-resolution rows my - 1, my, my + 1 (score channels)
    float* sc = smem_f + (size_t)3 * w * C;                        // [W][C] scores of one output row
    const int my = blockIdx.x, n = blockIdx.y, t = threadIdx.x;
    float* rows1 = smem_f;                                         // CPT = 1: [3][w][C]
    if constexpr (CPT == 1) {
        for (int i = t; i < 3 * w * C; i += kLabelThreads) {
            const int r = i / (w * C), j = i - r * (w * C);
            const int cell = j / C, c = j - cell * C;
            const int iy = min(max(my - 1 + r, 0), h - 1);
            rows1[i] = __ldg(lr + (((size_t)n * h + iy) * w + cell) * No + c);
        }
    } else {
        for (int i = t; i < 3 * w * C2; i += kLabelThreads) {
            const int r = i / (w * C2), j = i - r * (w * C2);
            const int cell = j / C2, c2 = j - cell * C2;
            const int iy = min(max(my - 1 + r, 0), h - 1);         // clamped like k_up8_heads; out-of-range rows get weight 0
            rows[i] = __ldg(reinterpret_cast<const float2*>(lr + (((size_t)n * h + iy) * w + cell) * No) + c2);
        }
    }
    __syncthreads();
    const float2 zero = make_float2(0.f, 0.f);
    for (int ty = 0; ty < 8; ty++) {
        const int y = 8 * my + ty;
        const int iy0 = ty < 4 ? my - 1 : my, iy1 = iy0 + 1;
        const float wy0 = (iy0 >= 0 && iy0 < h) ? deconv_w(y - 8 * iy0 + 4, 16) : 0.f;
        const float wy1 = (iy1 >= 0 && iy1 < h) ? deconv_w(y - 8 * iy1 + 4, 16) : 0.f;
        const float2* r0 = rows + (size_t)(iy0 - (my - 1)) * w * C2;     // staged slot of row iy0 (slot 0..2); clamping is
        const float2* r1 = rows + (size_t)(iy1 - (my - 1)) * w * C2;     // irrelevant where the weight is 0, identical otherwise
        if constexpr (CPT == 1) {
            const float* q0 = rows1 + (size_t)(iy0 - (my - 1)) * w * C;
            const float* q1 = rows1 + (size_t)(iy1 - (my - 1)) * w * C;
            for (int i = t; i < w * C; i += kLabelThreads) {
                const int mx = i / C, c = i - mx * C;
                const float bb = __ldg(bias_s + c);
                auto vb = [&](int cell) -> float { return up8_vblend(wy0, q0[cell * C + c], wy1, q1[cell * C + c]); };
                const float vl = mx > 0 ? vb(mx - 1) : 0.f;
                const float vc = vb(mx);
                const float vr = mx + 1 < w ? vb(mx + 1) : 0.f;
                float* sp = sc + (size_t)8 * mx * C + c;
#pragma unroll
                for (int tx = 0; tx < 8; tx++) {
                    const float wa = deconv_w(tx < 4 ? tx + 12 : tx + 4, 16), wb = deconv_w(tx < 4 ? tx + 4 : tx - 4, 16);
                    sp[tx * C] = fmaxf(up8_hblend(wa, tx < 4 ? vl : vc, wb, tx < 4 ? vc : vr, bb), 0.f);   // `score` has a ReLU
                }
            }
        } else {
            for (int i = t; i < w * C2; i += kLabelThreads) {
                const int mx = i / C2, c2 = i - mx * C2;
                const float2 bb = make_float2(__ldg(bias_s + 2 * c2), __ldg(bias_s + 2 * c2 + 1));
                auto vb = [&](int cell) -> float2 {
                    const float2 a = r0[cell * C2 + c2], b = r1[cell * C2 + c2];
                    return make_float2(up8_vblend(wy0, a.x, wy1, b.x), up8_vblend(wy0, a.y, wy1, b.y));
                };
                const float2 vl = mx > 0 ? vb(mx - 1) : zero;
                const float2 vc = vb(mx);
                const float2 vr = mx + 1 < w ? vb(mx + 1) : zero;
                float* sp = sc + (size_t)8 * mx * C + 2 * c2;
#pragma unroll
                for (int tx = 0; tx < 8; tx++) {
                    const float wa = deconv_w(tx < 4 ? tx + 12 : tx + 4, 16), wb = deconv_w(tx < 4 ? tx + 4 : tx - 4, 16);
                    const float2 a = tx < 4 ? vl : vc, b = tx < 4 ? vc : vr;
                    const float v0 = fmaxf(up8_hblend(wa, a.x, wb, b.x, bb.x), 0.f);      // `score` has a ReLU
                    const float v1 = fmaxf(up8_hblend(wa, a.y, wb, b.y, bb.y), 0.f);
                    *reinterpret_cast<float2*>(sp + tx * C) = make_float2(v0, v1);
                }
            }
        }
        __syncthreads();
        for (int x = t; x < W; x += kLabelThreads) {
            if constexpr (CPT == 1) {
                const float* s1 = sc + (size_t)x * C;
                float best = s1[0];
                int bi = 0;
                for (int c = 1; c < C; c++)
                    if (s1[c] > best) { best = s1[c]; bi = c; }
                label[((size_t)n * 8 * h + y) * W + x] = bi;
            } else {
                const float2* s2 = reinterpret_cast<const float2*>(sc + (size_t)x * C);
                float best = s2[0].x;
                int bi = 0;
                if (s2[0].y > best) { best = s2[0].y; bi = 1; }
                for (int c = 1; c < C2; c++) {
                    const float2 v = s2[c];
                    if (v.x > best) { best = v.x; bi = 2 * c; }
                    if (v.y > best) { best = v.y; bi = 2 * c + 1; }
                }
                label[((size_t)n * 8 * h + y) * W + x] = bi;
            }
        }
        __syncthreads();
    }
}

}  // namespace pcnn

using namespace pcnn;

extern "C" int pcnn_lowres_heads_nv(const void* score4, const void* score5, const void* vert4, const void* vert5,
                                    const float* w_score, const float* w_vertex, int B, int h, int w, int Cs, int Cv, int C,
                                    int num_vertex, float* out, void* stream)
{
    PCNN_REQUIRE(num_vertex == 3 * C || num_vertex == 0, "lowres_heads: num_vertex must be 3C or 0 (got %d, C = %d)", num_vertex, C);
    const bool vtx = num_vertex != 0;
    PCNN_REQUIRE(score4 && score5 && w_score && out && (!vtx || (vert4 && vert5)), "lowres_heads: NULL tensor pointer");
    PCNN_REQUIRE(vtx || (!vert4 && !vert5 && !w_vertex), "lowres_heads: the score-only head tensor takes no vertex tensors");
    const bool folded = vtx && w_vertex == nullptr;
    PCNN_REQUIRE(!folded || (3 * C <= Cv && Cv % 4 == 0), "lowres_heads: folded vertex head needs 3C <= Cv (got C = %d, Cv = %d)", C, Cv);
    PCNN_REQUIRE(h % 2 == 0 && w % 2 == 0, "lowres_heads: conv4 resolution must be even (got %d x %d)", h, w);
    if (vtx)
        PCNN_REQUIRE(Cs >= 4 && Cs % 4 == 0 && Cv % Cs == 0 && ((Cv / Cs) & (Cv / Cs - 1)) == 0,
                     "lowres_heads: need Cs %% 4 == 0 and Cv = 2^k Cs (got %d, %d)", Cs, Cv);
    else
        PCNN_REQUIRE(Cs >= 4 && Cs % 4 == 0, "lowres_heads: need Cs %% 4 == 0 (got %d)", Cs);
    PCNN_REQUIRE(C >= 1 && (!vtx || Cv / Cs <= 32), "lowres_heads: bad channel counts");
    size_t smem = sizeof(float) * (!vtx || folded ? (size_t)Cs * C + (size_t)kLrWarps * kLrPix * Cs
                                                  : (size_t)Cs * C + (size_t)Cv * 3 * C + (size_t)kLrWarps * kLrPix * (Cs + Cv));
    PCNN_REQUIRE(smem <= 200 * 1024, "lowres_heads: weights do not fit shared memory");
    auto kernel = vtx ? k_lowres_heads<true> : k_lowres_heads<false>;
    PCNN_SMEM_OPTIN(kernel, 200 * 1024, "lowres_heads");
    PCNN_REQUIRE((long long)B * h * w < 0x7fffffffLL, "lowres_heads: too many pixels");
    size_t npix = (size_t)B * h * w;
    int blocks = (int)std::min<size_t>((npix + kLrPix * kLrWarps - 1) / (kLrPix * kLrWarps), (size_t)kNumSMs * (vtx && !folded ? 2 : 8));
    kernel<<<blocks, 256, smem, (cudaStream_t)stream>>>((const __nv_bfloat16*)score4, (const __nv_bfloat16*)score5,
                                                        (const __nv_bfloat16*)vert4, (const __nv_bfloat16*)vert5, w_score, w_vertex, B, h,
                                                        w, Cs, Cv, C, out);
    return check_launch("lowres_heads");
}

extern "C" int pcnn_lowres_heads(const void* score4, const void* score5, const void* vert4, const void* vert5,
                                 const float* w_score, const float* w_vertex, int B, int h, int w, int Cs, int Cv, int C,
                                 float* out, void* stream)
{
    PCNN_REQUIRE(vert4 && vert5, "lowres_heads: NULL tensor pointer");
    return pcnn_lowres_heads_nv(score4, score5, vert4, vert5, w_score, w_vertex, B, h, w, Cs, Cv, C, 3 * C, out, stream);
}

// the launches of pcnn_up8_heads_nv for a head tensor of row stride 4C (kVertex) or C
template <bool kVertex>
static int up8_heads_launch(const float* lowres, const float* bias_score, const float* bias_vertex, int B, int h, int w, int C,
                            int32_t* label, float* vertex, float* prob, float* score, cudaStream_t stream)
{
    const bool odd = C % 2 != 0;   // odd C: the one-channel-per-thread forms (CPT = 1)
    if (!vertex && !prob && !score) {
        // label-only fast path: one CTA per low-resolution row (8 output rows), three staged rows + one score row in smem
        const size_t smem_l = sizeof(float) * ((size_t)3 * w * C + (size_t)8 * w * C);
        if (smem_l <= 200 * 1024 && h <= 65535) {
            dim3 grid_l(h, B);
            if (C == 22) {
                PCNN_SMEM_OPTIN((k_up8_label<22, 2, kVertex>), 200 * 1024, "up8_label<22>");
                k_up8_label<22, 2, kVertex><<<grid_l, kLabelThreads, smem_l, stream>>>(lowres, bias_score, h, w, C, label);
            } else if (odd) {
                PCNN_SMEM_OPTIN((k_up8_label<0, 1, kVertex>), 200 * 1024, "up8_label<0, odd>");
                k_up8_label<0, 1, kVertex><<<grid_l, kLabelThreads, smem_l, stream>>>(lowres, bias_score, h, w, C, label);
            } else {
                PCNN_SMEM_OPTIN((k_up8_label<0, 2, kVertex>), 200 * 1024, "up8_label<0>");
                k_up8_label<0, 2, kVertex><<<grid_l, kLabelThreads, smem_l, stream>>>(lowres, bias_score, h, w, C, label);
            }
            return check_launch("up8_label");
        }
    }
    const int No = (kVertex ? 4 : 1) * C;
    int seg_cells = w <= 20 ? w : 20;  // 160 output pixels per CTA
    size_t smem = sizeof(float) * ((size_t)(seg_cells + 2) * No + (size_t)8 * seg_cells * C + (size_t)16 * seg_cells);
    PCNN_REQUIRE(smem <= 200 * 1024, "up8_heads: segment does not fit shared memory (C = %d)", C);
    dim3 grid(8 * h, B, (w + seg_cells - 1) / seg_cells);
    PCNN_SMEM_OPTIN((k_up8_heads<0, 2, kVertex>), 200 * 1024, "up8_heads<0>");
    PCNN_SMEM_OPTIN((k_up8_heads<22, 2, kVertex>), 200 * 1024, "up8_heads<22>");
    PCNN_SMEM_OPTIN((k_up8_heads<0, 1, kVertex>), 200 * 1024, "up8_heads<0, odd>");
    if (C == 22)   // the YCB / LOV class count (lov_color_2d.yml:14): compile-time strides
        k_up8_heads<22, 2, kVertex><<<grid, 256, smem, stream>>>(lowres, bias_score, bias_vertex, h, w, C, seg_cells, label, vertex, prob,
                                                                 score);
    else if (odd)  // e.g. the multi-object LINEMOD model (linemod_color_2d.yml: 9 classes)
        k_up8_heads<0, 1, kVertex><<<grid, 256, smem, stream>>>(lowres, bias_score, bias_vertex, h, w, C, seg_cells, label, vertex, prob,
                                                                score);
    else
        k_up8_heads<0, 2, kVertex><<<grid, 256, smem, stream>>>(lowres, bias_score, bias_vertex, h, w, C, seg_cells, label, vertex, prob,
                                                                score);
    return check_launch("up8_heads");
}

extern "C" int pcnn_up8_heads_nv(const float* lowres, const float* bias_score, const float* bias_vertex, int B, int h, int w, int C,
                                 int num_vertex, int32_t* label, float* vertex, float* prob, float* score, void* stream)
{
    PCNN_REQUIRE(num_vertex == 3 * C || num_vertex == 0, "up8_heads: num_vertex must be 3C or 0 (got %d, C = %d)", num_vertex, C);
    // vertex == NULL: label-only mode (label_2d / prob / score; the dense vertex_pred is not produced)
    PCNN_REQUIRE(lowres && bias_score && label && (bias_vertex || !vertex), "up8_heads: NULL tensor pointer");
    PCNN_REQUIRE(num_vertex || (!vertex && !bias_vertex), "up8_heads: the score-only head tensor has no vertex channels");
    PCNN_REQUIRE(C >= 2 && C <= 128, "up8_heads: num_classes must be in 2..128 (got %d)", C);
    PCNN_REQUIRE(B >= 1 && h >= 1 && w >= 1, "up8_heads: bad shape");
    PCNN_REQUIRE(8 * h <= 65535 * 1 && B <= 65535, "up8_heads: image too tall for the launch grid");
    return num_vertex ? up8_heads_launch<true>(lowres, bias_score, bias_vertex, B, h, w, C, label, vertex, prob, score, (cudaStream_t)stream)
                      : up8_heads_launch<false>(lowres, bias_score, nullptr, B, h, w, C, label, nullptr, prob, score, (cudaStream_t)stream);
}

extern "C" int pcnn_up8_heads(const float* lowres, const float* bias_score, const float* bias_vertex, int B, int h, int w, int C,
                              int32_t* label, float* vertex, float* prob, float* score, void* stream)
{
    return pcnn_up8_heads_nv(lowres, bias_score, bias_vertex, B, h, w, C, 3 * C, label, vertex, prob, score, stream);
}
