// train_bwd.cu — the small kernels of the training step around the tensor-core GEMMs (csrc/wgrad_tc.cu, conv_tc.cu,
// fc_tc.cu): the un-fused FCN heads of the training graph and their gradients, the pose-loss chain, SGD with momentum.
//
// Training graph (lib/networks/vgg16_convs.py:128-212, lib/fcn/train.py:486-500), heads part:
//   add_score        = score_conv4 + up2(score_conv5)                  (deconv 4x4 / 2, fixed bilinear filter)
//   upscore -> score = relu(conv1x1(up8(add_score)) + b)  ==  relu(up8(conv1x1_nobias(add_score)) + b)   (commuted, heads.cu)
//   loss_cls         = -sum_{selected p} log_softmax(score)[p, gt_p] / count     (Hardlabel selection, train.py:455-465)
//   vertex_pred likewise from add_score_vertex; loss_vertex = smooth-L1 on the labelled pixels' own class (train.py:564-573)
// Backward pieces here:
//   k_up8_bwd_strip d lowres[b, my, mx, ch] = sum_{y, x} Wy Wx d up[b, y, x, ch]  with d up formed on the fly from the loss
//                   structure (one-hot cross-entropy through log-softmax and ReLU; sparse smooth-L1), never materialised
//   k_add_up2 / k_up2_bwd   add = a4 + up2(a5) and its adjoint (+ ReLU mask)
//   k_pose_chain_bwd        d fc8 pre-activation from Averagedistance's bottom_diff through l2_normalize, * weight, tanh
//   k_sgd_momentum          accum = mu * accum + g; w -= lr * accum (tf.train.MomentumOptimizer, train.py:633) + refreshed
//                           bf16 / fp16 tensor-core copy of the weights
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <float.h>

#include <type_traits>

#include "common.cuh"
#include "heads_common.cuh"

namespace pcnn {

// ---------------------------------------------------------------------------------------------
// add[b,h,w,c] = a4[b,h,w,c] + sum_i a5[b, i, j, c] * W4[h - 2 i + 1] * W4[w - 2 j + 1]   (conv2d_transpose 4x4 / 2, SAME)
// ---------------------------------------------------------------------------------------------
// thread = (pixel, group of 8 channels): 128-bit loads / stores (C % 8 == 0)
__device__ __forceinline__ void acc8(float acc[8], float wgt, const uint4& v)
{
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const float2 f = __bfloat1622float2(p[q]);
        acc[2 * q] = fmaf(wgt, f.x, acc[2 * q]);
        acc[2 * q + 1] = fmaf(wgt, f.y, acc[2 * q + 1]);
    }
}
__device__ __forceinline__ uint4 pack8(const float acc[8])
{
    uint4 o;
    __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int q = 0; q < 4; q++) p[q] = __floats2bfloat162_rn(acc[2 * q], acc[2 * q + 1]);
    return o;
}

__global__ void __launch_bounds__(256)
k_add_up2(const __nv_bfloat16* __restrict__ a4, const __nv_bfloat16* __restrict__ a5, int B, int h, int w, int C,
          __nv_bfloat16* __restrict__ out)
{
    const int h5 = h / 2, w5 = w / 2, cg = C / 8;
    const size_t total = (size_t)B * h * w * cg;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % cg);
        size_t r = i / cg;
        const int x = (int)(r % w); r /= w;
        const int y = (int)(r % h);
        const size_t n = r / h;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; q++) acc[q] = 0.f;
        acc8(acc, 1.f, __ldg(reinterpret_cast<const uint4*>(a4) + i));
        // contributing source rows: ky = y - 2 iy + 1 in [0, 4)
        for (int iy = (y - 2) / 2; iy <= (y + 1) / 2; iy++) {
            const int ky = y - 2 * iy + 1;
            if (iy < 0 || iy >= h5 || ky < 0 || ky >= 4) continue;
            for (int ix = (x - 2) / 2; ix <= (x + 1) / 2; ix++) {
                const int kx = x - 2 * ix + 1;
                if (ix < 0 || ix >= w5 || kx < 0 || kx >= 4) continue;
                acc8(acc, deconv_w(ky, 4) * deconv_w(kx, 4), __ldg(reinterpret_cast<const uint4*>(a5 + ((n * h5 + iy) * w5 + ix) * C) + g));
            }
        }
        reinterpret_cast<uint4*>(out)[i] = pack8(acc);
    }
}

// d a5[b, i, j, c] = [y5 > 0 or no relu] * sum_{y, x} W4[y - 2 i + 1] W4[x - 2 j + 1] d add[b, y, x, c]
__global__ void __launch_bounds__(256)
k_up2_bwd(const __nv_bfloat16* __restrict__ dadd /*[B,h,w,C]*/, const __nv_bfloat16* __restrict__ y5 /*[B,h/2,w/2,C] or null*/, int B,
          int h, int w, int C, __nv_bfloat16* __restrict__ d5)
{
    const int h5 = h / 2, w5 = w / 2, cg = C / 8;
    const size_t total = (size_t)B * h5 * w5 * cg;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % cg);
        size_t r = i / cg;
        const int ix = (int)(r % w5); r /= w5;
        const int iy = (int)(r % h5);
        const size_t n = r / h5;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; q++) acc[q] = 0.f;
        for (int ky = 0; ky < 4; ky++) {
            const int y = 2 * iy - 1 + ky;
            if (y < 0 || y >= h) continue;
            for (int kx = 0; kx < 4; kx++) {
                const int x = 2 * ix - 1 + kx;
                if (x < 0 || x >= w) continue;
                acc8(acc, deconv_w(ky, 4) * deconv_w(kx, 4), __ldg(reinterpret_cast<const uint4*>(dadd + ((n * h + y) * w + x) * C) + g));
            }
        }
        if (y5) {
            const uint4 yv = __ldg(reinterpret_cast<const uint4*>(y5) + i);
            const __nv_bfloat16* yp = reinterpret_cast<const __nv_bfloat16*>(&yv);
#pragma unroll
            for (int q = 0; q < 8; q++)
                if (!(__bfloat162float(yp[q]) > 0.f)) acc[q] = 0.f;
        }
        reinterpret_cast<uint4*>(d5)[i] = pack8(acc);
    }
}

// lowres [B,h,w,4C] f32 = [score part (first C of sc, row stride Cs) | vertex part (first 3C of vt, row stride Cv)];
// kVertex = false: the segmentation network's score-only [B,h,w,C] (vt not read)
template <bool kVertex>
__global__ void __launch_bounds__(256)
k_pack_lowres(const __nv_bfloat16* __restrict__ sc, int Cs, const __nv_bfloat16* __restrict__ vt, int Cv, size_t npix, int C,
              float* __restrict__ lowres)
{
    const int No = kVertex ? 4 * C : C;
    const size_t total = npix * No;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ch = (int)(i % No);
        const size_t p = i / No;
        lowres[i] = ch < C ? __bfloat162float(sc[p * Cs + ch]) : __bfloat162float(vt[p * Cv + ch - C]);
    }
}

// ---------------------------------------------------------------------------------------------
// k_up8_bwd_strip: gradient of both losses w.r.t. the low-resolution head tensor.
//   score channel c:  d up[p, c] = up_cls * sel_p * (prob[p, c] - [c == gt_p]) / (count + 1e-10) * [score[p, c] > 0]
//                     sel_p = gt_p != -1 and (gt_p > 0 or prob[p, gt_p] < threshold)          (Hardlabel, constant mask)
//   vertex channel 3c+k: pixels labelled c with a listed centre: up_vtx * w_inside * smoothL1'(w_inside (pred - target)) / (sum w + 1e-10)
// Outputs d lowres as TWO bf16 tensors in the layouts the 1x1 backward GEMMs read: d_sc [B,h,w,Cs] (first C channels,
// rest zero) and d_vt [B,h,w,Cv] (first 3C channels), plus per-CTA partial sums of d bias (the up-sampling weights of a
// pixel sum to the same value for bias: d b[ch] = sum_p d up[p, ch]).
// Organised so that every byte of prob / score is read (nearly) once and every load is coalesced.  CTA = (image, strip of SC
// low-resolution columns = 8 SC + 8 output columns incl. the halo, band of `rb` low-resolution rows).  Thread = (output column,
// channel PAIR): the CTA's threads read one contiguous run of (8 SC + 8) * C floats per output row of prob and of score (64-bit
// loads).  The thread walks DOWN the band's 8 rb + 8 output rows; a pixel row contributes to exactly two low-resolution rows (taps
// ky and ky + 8), so two running vertical sums per channel live in registers and the finished one is handed to the horizontal pass
// every 8 rows.  The three vertex channels of a labelled pixel go to a per-column shared-memory accumulator owned by the column's
// vertex-role thread (t < 8 SC + 8, below).  Bias gradients: per-thread registers (fixed channel pair) / per-column shared-memory
// cells, reduced over the columns in a fixed order (no atomics: run-to-run deterministic).
// Strip width SC: 4 cells for C >= 6 (40 columns x C / 2 pairs = 120 .. 1000 threads).  At C = 2 a column is one thread, so a 4-cell
// strip would be a 40-thread CTA; the two-class kernel takes 16 cells (136 threads), which also cuts the halo.
// Redundant reads: (8 SC + 8) / (8 SC) x (8 rb + 8) / (8 rb) = 1.25 x 1.07 at SC = 4, 1.06 x 1.07 at SC = 16 (rb = 16).
// CPT = channels per thread: 2 (C even, the pairs above) or 1 (C = 9: a pixel's score / prob row is not 8-byte aligned, so a thread
// owns (output column, channel), kSCols * C threads with one running (lo, hi, bias) triple and 32-bit loads; the CTA still reads
// one contiguous run of (8 SC + 8) * C floats per output row).
// ---------------------------------------------------------------------------------------------
constexpr int kStrip = 4;                           // strip width (cells) of the C >= 6 kernels
constexpr int kStrip2 = 16;                         // strip width (cells) of the C = 2 kernel
constexpr int kBand = 16;                           // band height (low-resolution rows) of every CTA

// Target mode kCoord (VERTEX_REG_3D): the vertex target is the pixel's object coordinate vertmap [B,H,W,3] scaled by its class's
// extents (coord_scale / coord_target, heads_common.cuh) instead of the 2-D centre direction + log z.  The per-class (a_k, b_k) sit in
// shared memory after the per-class listed flags (where the 2-D mode keeps log z: 6 C more floats), and the vertex-role thread loads
// a pixel's three vertmap floats one row ahead, together with the label it already prefetches, and only for weighted pixels.
// C = 2: 6 resident CTAs per SM caps the kernel at 64 registers without spills in the 2-D mode (-Xptxas -v; the 3-D mode spills a few
// bytes, DESIGN §10); 8 would spill.
// CPT = 1 runs at C = 9 only (kSCols * 9 = 360 threads): bounding it at 360 x 2 CTAs instead of 1024 lifts the register cap from 64,
// where the coordinate form spills, to 80
// kVertex = false: target mode "none", the segmentation network's adjoint of loss_cls alone (no vertex head): no vertex-role work and no
// vacc / bv / logz / ab shared memory; vertex_loss_out, lowres, bias_v, centers, vertmap, extents and d_vt are not read, and a CTA's
// dbias_partial row holds C floats instead of 4C.  The score channels' arithmetic is the vertex modes' own, so d_sc and the score
// bias gradient equal theirs bit for bit.
template <int CT, int SC, bool kCoord, int CPT, bool kVertex>
__global__ void __launch_bounds__(CT ? (8 * SC + 8) * (CT / 2) : (CPT == 1 ? (8 * SC + 8) * 9 : 1024), CT == 2 ? 6 : (CT || CPT == 1 ? 2 : 1))
k_up8_bwd_strip(const float* __restrict__ prob, const float* __restrict__ score, const int* __restrict__ gt, const float* __restrict__ cls_out,
                float up_cls, float threshold, const float* __restrict__ lowres,
                const float* __restrict__ bias_v, const float* __restrict__ centers,
                const float* __restrict__ vtx_out, float up_vtx, float w_inside, float sigma2, int h, int w, int rb, int C_rt, int Cs, int Cv,
                __nv_bfloat16* __restrict__ d_sc, __nv_bfloat16* __restrict__ d_vt, float* __restrict__ dbias_partial /*[ctas][4C or C]*/,
                const float* __restrict__ vertmap, const float* __restrict__ extents)
{
    // C == 2 or C even in 6..50: thread = (output column, channel pair), kSCols * C / 2 threads; C = 9: (output column, channel),
    // kSCols * C threads.  Threads t < kSCols also own the vertex channels of output column t (at C = 2 that is every thread)
    using V = std::conditional_t<CPT == 2, float2, float>;
    constexpr int kSC = SC, kSCols = 8 * SC + 8;
    const int C = CT ? CT : C_rt;
    const int CP = C / CPT, No = 4 * C, VC = 3 * C, NT = kSCols * CP;
    const int H = 8 * h, W = 8 * w;
    const int c_lo = blockIdx.x * kSC, c_hi = min(c_lo + kSC, w);
    const int m_lo = blockIdx.y * rb, m_hi = min(m_lo + rb, h);
    const int n = blockIdx.z;
    const float s_cls = up_cls / (cls_out[1] + 1e-10f), s_vtx = kVertex ? up_vtx / (vtx_out[1] + 1e-10f) : 0.f;
    const size_t img = (size_t)n * H * W;
    extern __shared__ float sm[];
    float* v_s = sm;                                 // [kSCols][C]       finished vertical sums of the score channels
    float* vacc = v_s + kSCols * C;                  // [2][kSCols][VC]   running vertical sums of the vertex channels
    float* bs = vacc + (kVertex ? 2 * kSCols * VC : 0);   // [kSCols][C]  bias-gradient sums (score), per column
    float* bv = bs + kSCols * C;                     // [kSCols][VC]      bias-gradient sums (vertex), per column
    float* logz = bv + kSCols * VC;                  // [C]               log of the listed centre depth of each class of this image
                                                     //                   (kCoord: 1 if the class is listed, else 0)
    float* ab = logz + C;                            // [C][6]            kCoord: (a_0, b_0, a_1, b_1, a_2, b_2) of each class
    const int t = threadIdx.x, col = t / CP, j = t - col * CP;
    if constexpr (kVertex) {
        for (int i = t; i < C; i += NT) {
            const float z = centers[((size_t)n * C + i) * 3 + 2];
            if constexpr (kCoord) {
                logz[i] = z > 0.f ? 1.f : 0.f;
                coord_scale(extents + 3 * i, ab + 6 * i);
            } else {
                logz[i] = z > 0.f ? (float)log((double)z) : 0.f;
            }
        }
        for (int i = t; i < 2 * kSCols * VC; i += NT) vacc[i] = 0.f;
        for (int i = t; i < kSCols * VC; i += NT) bv[i] = 0.f;
    }
    __syncthreads();
    const int x = 8 * c_lo - 4 + col;
    const bool xin = x >= 0 && x < W && x < 8 * c_hi + 4;
    const bool own_x = x >= 8 * c_lo && x < 8 * c_hi;
    float lo0 = 0.f, lo1 = 0.f, hi0 = 0.f, hi1 = 0.f, b0 = 0.f, b1 = 0.f;
    int slot_lo = 0;                                 // vacc half of the OLDER low-resolution row (taps 8..15)
    const int y_end = 8 * (m_hi - 1) + 11;
    // Three-stage software pipeline over the rows (the loads of a row depend on its label: label -> selected? -> score / prob pair):
    // row y + 2: label + background probability in flight; row y + 1: label known, its score / prob pair in flight; row y: consumed.
    // Hardlabel selects a background pixel only if prob[.., 0] < threshold and every foreground pixel, so the one probability the
    // selection needs is channel 0 — independent of the label's value, loaded together with it.
    // Addressing: per-thread base pointers at (image n, row 0, column x) and ONE 32-bit pixel-row offset `ro` advanced by W per row
    // (the first version recomputed `img + y W + x` in 64 bits for every load: 135 instructions per row, 9 % of them loads or math).
    const int y_first = max(8 * m_lo - 4, 0);        // rows above the image contribute nothing and complete no low-resolution row
    const int y_last = min(y_end, H - 1);            // last row with pixels; the loop runs to y_end for the final hand-over
    const int xs = xin ? x : 0;                      // a thread outside the strip / image never loads (labels stay -1)
    const int* gt_c = gt + img + xs;
    const float* pr0_c = prob + (img + xs) * C;
    const V* sc2_c = reinterpret_cast<const V*>(score) + (img + xs) * CP + j;
    const V* pr2_c = reinterpret_cast<const V*>(prob) + (img + xs) * CP + j;
    const int j2 = CPT * j;
    const int own_lo = 8 * m_lo, own_hi = 8 * m_hi;
    // vertex role (threads t < kSCols): column xB, labels prefetched two rows ahead
    const int xB = 8 * c_lo - 4 + t;
    const bool xinB = t < kSCols && xB >= 0 && xB < W && xB < 8 * c_hi + 4;
    const bool ownB_x = xB >= 8 * c_lo && xB < 8 * c_hi;
    const int* gtB_c = gt + img + (xinB ? xB : 0);
    // running pointers, advanced by one image row per iteration: labels / background probability two rows ahead, score / prob pair one
    // row ahead (pointer bumps keep the loop body free of 64-bit index multiplications)
    const size_t r0 = (size_t)y_first * W;
    const int* gp2 = gt_c + r0 + 2 * (size_t)W;
    const float* qp2 = pr0_c + (r0 + 2 * (size_t)W) * C;
    const V* sp1 = sc2_c + (r0 + W) * CP;
    const V* pp1 = pr2_c + (r0 + W) * CP;
    const int* gpB2 = gtB_c + r0 + 2 * (size_t)W;
    const size_t stepQ = (size_t)W * C, stepS = (size_t)W * CP;
    int gB0 = -1, gB1 = -1;
    if (kVertex && xinB) {
        if (y_first <= y_last) gB0 = __ldg(gtB_c + r0);
        if (y_first + 1 <= y_last) gB1 = __ldg(gtB_c + r0 + W);
    }
    // kCoord: object coordinate of the vertex-role pixel of the current row, loaded one row ahead for weighted pixels only
    float vB[3] = {0.f, 0.f, 0.f};
    if constexpr (kCoord && kVertex) {
        if (gB0 > 0 && gB0 < C && logz[gB0] > 0.f) {
            const float* vp = vertmap + (img + r0 + xB) * 3;
            vB[0] = __ldg(vp); vB[1] = __ldg(vp + 1); vB[2] = __ldg(vp + 2);
        }
    }
    int g0 = -1, g1 = -1, g2;
    float q0 = 0.f, q1 = 0.f, q2;
    V sv0 = V{}, pv0 = sv0, sv1 = sv0, pv1 = sv0;
    if (xin) {
        if (y_first <= y_last) { g0 = __ldg(gt_c + r0); q0 = __ldg(pr0_c + r0 * C); }
        if (y_first + 1 <= y_last) { g1 = __ldg(gt_c + r0 + W); q1 = __ldg(pr0_c + (r0 + W) * C); }
    }
    bool s0 = (unsigned)g0 < (unsigned)C && (g0 > 0 || q0 < threshold);
    if (s0) { sv0 = __ldg(sc2_c + r0 * CP); pv0 = __ldg(pr2_c + r0 * CP); }
    for (int y = y_first; y <= y_end; y++) {
        const int kh = (y + 4) & 7;                  // tap of the newer row m_new = (y + 4) >> 3; the older row m_new - 1 sees tap kh + 8
        const float w_hi = 1.f - fabsf((float)kh * 0.125f - 0.9375f), w_lo = 1.f - fabsf((float)(kh + 8) * 0.125f - 0.9375f);   // deconv_w(., 16)
        g2 = -1; q2 = 0.f;
        if (xin && y + 2 <= y_last) { g2 = __ldg(gp2); q2 = __ldg(qp2); }
        const bool s1 = (unsigned)g1 < (unsigned)C && (g1 > 0 || q1 < threshold);
        if (s1) { sv1 = __ldg(sp1); pv1 = __ldg(pp1); }
        gp2 += W; qp2 += stepQ; sp1 += stepS; pp1 += stepS;
        if constexpr (CPT == 1) {
            if (s0) {
                const float d0 = sv0 > 0.f ? s_cls * (pv0 - (j == g0 ? 1.f : 0.f)) : 0.f;
                lo0 = fmaf(w_lo, d0, lo0);
                hi0 = fmaf(w_hi, d0, hi0);
                if (own_x && y >= own_lo && y < own_hi) b0 += d0;
            }
        } else if (s0) {
            const float d0 = sv0.x > 0.f ? s_cls * (pv0.x - (j2 == g0 ? 1.f : 0.f)) : 0.f;
            const float d1 = sv0.y > 0.f ? s_cls * (pv0.y - (j2 + 1 == g0 ? 1.f : 0.f)) : 0.f;
            lo0 = fmaf(w_lo, d0, lo0); lo1 = fmaf(w_lo, d1, lo1);
            hi0 = fmaf(w_hi, d0, hi0); hi1 = fmaf(w_hi, d1, hi1);
            if (own_x && y >= own_lo && y < own_hi) { b0 += d0; b1 += d1; }
        }
        // ---- vertex role: thread t < kSCols owns output column t of the strip (all three vertex channels of the pixel's class).
        // The target direction needs a double sqrt and two double divisions per labelled pixel (the reference forms it in float64,
        // minibatch.py:582-594); keeping that on kSCols densely packed lanes instead of three lanes of every column costs 1/7 of the
        // double-precision issue slots at C = 22 (the (column, k) mapping made the whole kernel FP64-bound: 3.2 ms at batch 64).
        if (kVertex && t < kSCols) {
            const int gB = gB0;
            if (gB > 0 && gB < C) {
                const float* cen = centers + ((size_t)n * C + gB) * 3;
                if (kCoord ? logz[gB] > 0.f : cen[2] > 0.f) {
                    const bool ownB = ownB_x && y >= own_lo && y < own_hi;
                    float tg[3];
                    if constexpr (kCoord) {
                        const float* s = ab + 6 * gB;
#pragma unroll
                        for (int k = 0; k < 3; k++) tg[k] = coord_target(s[2 * k], s[2 * k + 1], vB[k]);
                    } else {
                        const double dx = (double)cen[0] - (double)xB, dy = (double)cen[1] - (double)y;
                        const double nrm = sqrt(dx * dx + dy * dy) + 1e-10;
                        tg[0] = (float)(dx / nrm); tg[1] = (float)(dy / nrm); tg[2] = logz[gB];
                    }
                    float* a_lo = vacc + ((size_t)slot_lo * kSCols + t) * VC + 3 * gB;
                    float* a_hi = vacc + ((size_t)(slot_lo ^ 1) * kSCols + t) * VC + 3 * gB;
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        // vertex_pred's value, formed from the low-resolution head tensor with k_up8_heads' operation sequence
                        const float pv = up8_value(lowres, n, h, w, No, C + 3 * gB + k, y, xB, __ldg(bias_v + 3 * gB + k));
                        const float diff = w_inside * (pv - tg[k]);
                        const float ad = fabsf(diff);
                        const float dt = ad < 1.f / sigma2 ? diff * sigma2 : (diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f));
                        const float d = s_vtx * w_inside * dt;
                        a_lo[k] = fmaf(w_lo, d, a_lo[k]);
                        a_hi[k] = fmaf(w_hi, d, a_hi[k]);
                        if (ownB) bv[t * VC + 3 * gB + k] += d;
                    }
                }
            }
            gB0 = gB1;
            gB1 = (xinB && y + 2 <= y_last) ? __ldg(gpB2) : -1;
            gpB2 += W;
            if constexpr (kCoord) {
                if (gB0 > 0 && gB0 < C && logz[gB0] > 0.f) {   // a label >= 0 is only ever loaded for rows <= y_last
                    const float* vp = vertmap + (img + (size_t)(y + 1) * W + xB) * 3;
                    vB[0] = __ldg(vp); vB[1] = __ldg(vp + 1); vB[2] = __ldg(vp + 2);
                }
            }
        }
        g0 = g1; q0 = q1; s0 = s1; sv0 = sv1; pv0 = pv1; g1 = g2; q1 = q2;
        if (kh == 7) {
            // the older row m_old = ((y + 4) >> 3) - 1 has seen its last tap (15)
            const int m_old = ((y + 4) >> 3) - 1;
            if (m_old >= m_lo) {                      // block-uniform (m_old < m_hi by the loop bounds)
                if constexpr (CPT == 1) v_s[col * C + j] = lo0;
                else { v_s[col * C + 2 * j] = lo0; v_s[col * C + 2 * j + 1] = lo1; }
            }
            __syncthreads();                          // every thread's updates of vacc for this row are done (also when the row is discarded)
            if (m_old >= m_lo) {
                const float* va = vacc + (size_t)slot_lo * kSCols * VC;
                const int Ct = kVertex ? Cs + Cv : Cs;   // channels of a d_sc (+ d_vt) cell
                for (int item = t; item < (c_hi - c_lo) * Ct; item += NT) {
                    const int ml = item / Ct, ch = item - ml * Ct;
                    const size_t cell = ((size_t)n * h + m_old) * w + c_lo + ml;
                    float acc = 0.f;
                    if (ch < Cs) {
                        if (ch < C) {
#pragma unroll
                            for (int kx = 0; kx < 16; kx++) acc = fmaf(deconv_w(kx, 16), v_s[(8 * ml + kx) * C + ch], acc);
                        }
                        d_sc[cell * Cs + ch] = __float2bfloat16_rn(acc);
                    } else {
                        const int c2 = ch - Cs;
                        if (c2 < VC) {
#pragma unroll
                            for (int kx = 0; kx < 16; kx++) acc = fmaf(deconv_w(kx, 16), va[(8 * ml + kx) * VC + c2], acc);
                        }
                        d_vt[cell * Cv + c2] = __float2bfloat16_rn(acc);
                    }
                }
                __syncthreads();
            }
            if constexpr (kVertex)
                for (int i = t; i < kSCols * VC; i += NT) vacc[(size_t)slot_lo * kSCols * VC + i] = 0.f;
            __syncthreads();
            lo0 = hi0; lo1 = hi1; hi0 = 0.f; hi1 = 0.f;
            slot_lo ^= 1;
        }
    }
    if constexpr (CPT == 1) bs[col * C + j] = b0;
    else { bs[col * C + 2 * j] = b0; bs[col * C + 2 * j + 1] = b1; }
    __syncthreads();
    const size_t cta = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    const int NB = kVertex ? No : C;                 // bias channels
    for (int ch = t; ch < NB; ch += NT) {
        float acc = 0.f;
        if (ch < C) { for (int q = 0; q < kSCols; q++) acc += bs[q * C + ch]; }
        else { for (int q = 0; q < kSCols; q++) acc += bv[q * VC + ch - C]; }
        dbias_partial[cta * NB + ch] = acc;
    }
}

// out[i] = scale * sum_k partial[k][i] (+ decay * p[i]); block = 32 columns x 8 row groups, groups combined in fixed order
__global__ void __launch_bounds__(256)
k_sum_partials(const float* __restrict__ partial, int nparts, int n, float scale, const float* __restrict__ p, float decay, float* __restrict__ out)
{
    __shared__ float s[8][33];
    const int cl = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + cl;
    float acc = 0.f;
    if (i < n)
        for (int k = grp; k < nparts; k += 8) acc += partial[(size_t)k * n + i];
    s[grp][cl] = acc;
    __syncthreads();
    if (grp == 0 && i < n) {
        float t = 0.f;
#pragma unroll
        for (int q = 0; q < 8; q++) t += s[q][cl];
        t *= scale;
        if (p) t = fmaf(decay, p[i], t);
        out[i] = t;
    }
}

// ---------------------------------------------------------------------------------------------
// pose chain (vgg16_convs.py:195-200): poses_pred = l2_normalize(poses_tanh * poses_weight, dim 1); loss = Averagedistance.
// g = upstream * bottom_diff [N,4C];  u = tanh * w;  nrm = sqrt(max(sum u^2, 1e-12));  p = u / nrm;
// d u = (g - p (p . g)) / nrm (zero where the clamp is active);  d pre = d u * w * (1 - tanh^2).   One warp per row.
// Output fp16 [N, ld] (the fc8 backward GEMMs' operand), padding columns zero.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_pose_chain_bwd(const float* __restrict__ g, const float* __restrict__ tanhv, const float* __restrict__ wgt, int N, int D, float upstream,
                 __half* __restrict__ dpre, int ld)
{
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= N) return;
    float su = 0.f, sg = 0.f;
    for (int j = lane; j < D; j += 32) {
        const float u = tanhv[(size_t)row * D + j] * wgt[(size_t)row * D + j];
        su = fmaf(u, u, su);
        sg = fmaf(u, upstream * g[(size_t)row * D + j], sg);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { su += __shfl_xor_sync(0xffffffffu, su, o); sg += __shfl_xor_sync(0xffffffffu, sg, o); }
    const bool clamped = su < 1e-12f;
    const float inv = rsqrtf(fmaxf(su, 1e-12f));
    for (int j = lane; j < ld; j += 32) {
        float d = 0.f;
        if (j < D) {
            const float t = tanhv[(size_t)row * D + j], wv = wgt[(size_t)row * D + j];
            const float u = t * wv, gg = upstream * g[(size_t)row * D + j];
            // p = u * inv; d u = (g - p (p.g)) * inv, (p.g) = sg * inv; with the clamp active the norm is the constant 1e-6
            const float du = clamped ? gg * inv : (gg - u * inv * (sg * inv)) * inv;
            d = du * wv * (1.f - t * t);
        }
        dpre[(size_t)row * ld + j] = __float2half_rn(sat_f16(d));
    }
}

// ---------------------------------------------------------------------------------------------
// SGD with momentum on fp32 master weights + the refreshed 16-bit tensor-core copy
// ---------------------------------------------------------------------------------------------
template <typename T16>
__device__ __forceinline__ T16 to16(float v);
template <>
__device__ __forceinline__ __nv_bfloat16 to16<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <>
__device__ __forceinline__ __half to16<__half>(float v) { return __float2half_rn(sat_f16(v)); }

template <typename T16>
__global__ void __launch_bounds__(256)
k_sgd_momentum(float* __restrict__ w, float* __restrict__ accum, const float* __restrict__ grad, size_t n, float lr, float mu, float wd,
               float gscale, T16* __restrict__ copy16)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        // gradient of loss + wd * |w|^2 / 2 (l2_regularizer on weights and biases, network.py:171-172, 184)
        const float a = fmaf(mu, accum[i], fmaf(wd, w[i], gscale * grad[i]));
        accum[i] = a;
        const float v = fmaf(-lr, a, w[i]);
        w[i] = v;
        if (copy16) copy16[i] = to16<T16>(v);
    }
}

// out[c][r] = in[r][c] (16-bit elements), tiled through shared memory: the [in][out] copy of a fully connected weight
// matrix for its input-gradient GEMM
__global__ void __launch_bounds__(256)
k_transpose16(const uint16_t* __restrict__ in, int rows, int cols, uint16_t* __restrict__ out)
{
    __shared__ uint16_t tile[64][66];
    const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int r = i / 64, c = i % 64;
        tile[r][c] = (r0 + r < rows && c0 + c < cols) ? in[(size_t)(r0 + r) * cols + c0 + c] : (uint16_t)0;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int c = i / 64, r = i % 64;
        if (c0 + c < cols && r0 + r < rows) out[(size_t)(c0 + c) * rows + r0 + r] = tile[r][c];
    }
}

// 16-bit conversions of small gradient tensors (fp16 <-> bf16 <-> f32): dst[i] = (T)src[i]
__global__ void __launch_bounds__(256)
k_half_to_float(const __half* __restrict__ src, size_t n, float scale, float* __restrict__ dst)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = scale * __half2float(src[i]);
}

}  // namespace pcnn

using namespace pcnn;

static int ew_blocks(size_t total) { return (int)std::min<size_t>((total + 255) / 256, (size_t)kNumSMs * 8); }

extern "C" int pcnn_add_up2_bf16(const void* a4, const void* a5, int B, int h, int w, int C, void* out, void* stream)
{
    PCNN_REQUIRE(a4 && a5 && out && h % 2 == 0 && w % 2 == 0 && C % 8 == 0, "add_up2: bad arguments (even h, w; C %% 8 == 0)");
    k_add_up2<<<ew_blocks((size_t)B * h * w * (C / 8)), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)a4, (const __nv_bfloat16*)a5, B, h, w, C,
                                                                                (__nv_bfloat16*)out);
    return check_launch("add_up2");
}

extern "C" int pcnn_up2_bwd_bf16(const void* dadd, const void* y5, int B, int h, int w, int C, void* d5, void* stream)
{
    PCNN_REQUIRE(dadd && d5 && h % 2 == 0 && w % 2 == 0 && C % 8 == 0, "up2_bwd: bad arguments (even h, w; C %% 8 == 0)");
    k_up2_bwd<<<ew_blocks((size_t)B * (h / 2) * (w / 2) * (C / 8)), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dadd, (const __nv_bfloat16*)y5, B, h,
                                                                                            w, C, (__nv_bfloat16*)d5);
    return check_launch("up2_bwd");
}

extern "C" int pcnn_pack_lowres_nv(const void* sc, int Cs, const void* vt, int Cv, int B, int h, int w, int C, int num_vertex, float* lowres,
                                   void* stream)
{
    PCNN_REQUIRE(num_vertex == 3 * C || num_vertex == 0, "pack_lowres: num_vertex must be 3C or 0 (got %d, C = %d)", num_vertex, C);
    const bool vtx = num_vertex != 0;
    PCNN_REQUIRE(sc && lowres && Cs >= C && (vtx ? vt && Cv >= 3 * C : !vt), "pack_lowres: bad arguments");
    const size_t npix = (size_t)B * h * w;
    const int blocks = ew_blocks(npix * (vtx ? 4 : 1) * C);
    if (vtx)
        k_pack_lowres<true><<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)sc, Cs, (const __nv_bfloat16*)vt, Cv, npix, C, lowres);
    else
        k_pack_lowres<false><<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)sc, Cs, nullptr, 0, npix, C, lowres);
    return check_launch("pack_lowres");
}

extern "C" int pcnn_pack_lowres(const void* sc, int Cs, const void* vt, int Cv, int B, int h, int w, int C, float* lowres, void* stream)
{
    PCNN_REQUIRE(vt, "pack_lowres: bad arguments");
    return pcnn_pack_lowres_nv(sc, Cs, vt, Cv, B, h, w, C, 3 * C, lowres, stream);
}

// CTAs of k_up8_bwd_strip: (image, strip of cells, band of kBand rows); each writes one row of bias partial sums
static size_t up8_bwd_ctas(int B, int h, int w, int C)
{
    const int sc = C == 2 ? kStrip2 : kStrip;
    return (size_t)B * ((w + sc - 1) / sc) * ((h + kBand - 1) / kBand);
}

extern "C" int pcnn_up8_heads_bwd_workspace_bytes(int B, int h, int w, int C, size_t* bytes)
{
    PCNN_REQUIRE(bytes && B >= 1 && h >= 1 && w >= 1 && C >= 1, "up8_heads_bwd_workspace_bytes: bad arguments");
    // partial bias sums of k_up8_bwd_strip: one row of 4C floats per CTA
    *bytes = sizeof(float) * up8_bwd_ctas(B, h, w, C) * 4 * C;
    return PCNN_OK;
}

extern "C" int pcnn_up8_scores_bwd_workspace_bytes(int B, int h, int w, int C, size_t* bytes)
{
    PCNN_REQUIRE(bytes && B >= 1 && h >= 1 && w >= 1 && C >= 1, "up8_scores_bwd_workspace_bytes: bad arguments");
    // partial bias sums of k_up8_bwd_strip in target mode "none": one row of C floats per CTA
    *bytes = sizeof(float) * up8_bwd_ctas(B, h, w, C) * C;
    return PCNN_OK;
}

// every instantiation of the strip kernel has this signature; the launch picks one by class count and target mode
using UpBwdKernel = decltype(&k_up8_bwd_strip<2, kStrip2, false, 2, true>);
enum UpBwdTarget { kTarget2D, kTargetCoord, kTargetNone };
template <int CT, int SC, int CPT>
static UpBwdKernel up8_bwd_kernel(UpBwdTarget target)
{
    return target == kTargetNone ? k_up8_bwd_strip<CT, SC, false, CPT, false>
                                 : (target == kTargetCoord ? k_up8_bwd_strip<CT, SC, true, CPT, true> : k_up8_bwd_strip<CT, SC, false, CPT, true>);
}

// the shared tail of pcnn_up8_heads_bwd and pcnn_up8_scores_bwd (arguments validated by the caller)
static int up8_bwd_launch(UpBwdTarget target, const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out,
                          float upstream_cls, float threshold, const float* lowres, const float* bias_vertex, const float* centers,
                          const float* vertmap, const float* extents, const float* vertex_loss_out, float upstream_vertex, float w_inside,
                          float sigma, int B, int h, int w, int C, int Cs, int Cv, void* d_sc_bf16, void* d_vt_bf16, float* dbias,
                          void* workspace, void* stream)
{
    // coalesced strip kernel (see k_up8_bwd_strip)
    const int sc = C == 2 ? kStrip2 : kStrip, cols = 8 * sc + 8;
    const int bands = (h + kBand - 1) / kBand, strips = (w + sc - 1) / sc;
    PCNN_REQUIRE(bands <= 65535, "up8_heads_bwd: bad shape");
    UpBwdKernel kernel;
    int threads;
    if (C == 22) {
        kernel = up8_bwd_kernel<22, kStrip, 2>(target);
        threads = cols * 11;
    } else if (C == 2) {
        kernel = up8_bwd_kernel<2, kStrip2, 2>(target);
        threads = cols;
    } else if (C % 2) {   // C = 9: one channel per thread (at 40 x 9 threads the strip's shared memory is 16 KB: no opt-in)
        kernel = up8_bwd_kernel<0, kStrip, 1>(target);
        threads = cols * C;
    } else {
        kernel = up8_bwd_kernel<0, kStrip, 2>(target);
        threads = cols * (C / 2);
        PCNN_SMEM_OPTIN(kernel, 100 * 1024,
                        target == kTargetNone ? "up8_bwd_strip<0, none>" : (target == kTargetCoord ? "up8_bwd_strip<0, coord>" : "up8_bwd_strip<0>"));
    }
    cudaStream_t st = (cudaStream_t)stream;
    // score-only: v_s + bs ([kSCols][C] each); vertex modes add vacc, bv, logz (and the 3-D mode's ab)
    const size_t smem = sizeof(float) * (target == kTargetNone ? (size_t)cols * 2 * C
                                                               : (size_t)cols * 11 * C + C + (target == kTargetCoord ? 6 * C : 0));
    kernel<<<dim3(strips, bands, B), threads, smem, st>>>(prob, score, gt, cls_loss_out, upstream_cls, threshold, lowres, bias_vertex, centers,
                                                          vertex_loss_out, upstream_vertex, w_inside, sigma * sigma, h, w, kBand, C, Cs, Cv,
                                                          (__nv_bfloat16*)d_sc_bf16, (__nv_bfloat16*)d_vt_bf16, (float*)workspace, vertmap,
                                                          extents);
    const int nb = target == kTargetNone ? C : 4 * C;
    k_sum_partials<<<(nb + 31) / 32, 256, 0, st>>>((const float*)workspace, B * strips * bands, nb, 1.f, nullptr, 0.f, dbias);
    return check_launch("up8_heads_bwd");
}

// the target mode follows vertmap / extents: both NULL = 2-D centre direction, both given = 3-D object coordinate (VERTEX_REG_3D:
// vertmap [B,8h,8w,3] f32 and extents [C,3] f32; centers stays the presence table, a class's pixels are weighted iff
// centers[b, c, 2] > 0)
extern "C" int pcnn_up8_heads_bwd(const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out, float upstream_cls,
                                  float threshold, const float* lowres, const float* bias_vertex, const float* centers, const float* vertmap,
                                  const float* extents, const float* vertex_loss_out, float upstream_vertex, float w_inside, float sigma, int B,
                                  int h, int w, int C, int Cs, int Cv, void* d_sc_bf16, void* d_vt_bf16, float* dbias, void* workspace,
                                  size_t workspace_bytes, void* stream)
{
    PCNN_REQUIRE(prob && score && gt && cls_loss_out && lowres && bias_vertex && centers && vertex_loss_out && d_sc_bf16 && d_vt_bf16 &&
                     dbias && workspace,
                 "up8_heads_bwd: NULL tensor pointer");
    PCNN_REQUIRE(!vertmap == !extents, "up8_heads_bwd: vertmap and extents must both be given (3-D target) or both be NULL (2-D target)");
    PCNN_REQUIRE(Cs >= C && Cv >= 3 * C && h <= 65535 && B <= 65535, "up8_heads_bwd: bad shape");
    // class counts of the reference's configurations: 2 (single object), 22 (YCB), 9 (multi-object LINEMOD), and the even range
    PCNN_REQUIRE(C == 2 || C == 9 || (C % 2 == 0 && C >= 6 && C <= 50), "up8_heads_bwd: C must be even and 2 or in 6..50, or 9 (C = %d)", C);
    size_t need = 0;
    PCNN_REQUIRE(pcnn_up8_heads_bwd_workspace_bytes(B, h, w, C, &need) == PCNN_OK, "up8_heads_bwd: bad shape");
    PCNN_REQUIRE(workspace_bytes >= need, "up8_heads_bwd: workspace too small (%zu < %zu)", workspace_bytes, need);
    return up8_bwd_launch(vertmap ? kTargetCoord : kTarget2D, prob, score, gt, cls_loss_out, upstream_cls, threshold, lowres, bias_vertex,
                          centers, vertmap, extents, vertex_loss_out, upstream_vertex, w_inside, sigma, B, h, w, C, Cs, Cv, d_sc_bf16,
                          d_vt_bf16, dbias, workspace, stream);
}

extern "C" int pcnn_up8_scores_bwd(const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out, float upstream_cls,
                                   float threshold, int B, int h, int w, int C, int Cs, void* d_sc_bf16, float* dbias, void* workspace,
                                   size_t workspace_bytes, void* stream)
{
    PCNN_REQUIRE(prob && score && gt && cls_loss_out && d_sc_bf16 && dbias && workspace, "up8_scores_bwd: NULL tensor pointer");
    PCNN_REQUIRE(Cs >= C && h <= 65535 && B <= 65535, "up8_scores_bwd: bad shape");
    PCNN_REQUIRE(C == 2 || C == 9 || (C % 2 == 0 && C >= 6 && C <= 50), "up8_scores_bwd: C must be even and 2 or in 6..50, or 9 (C = %d)", C);
    size_t need = 0;
    PCNN_REQUIRE(pcnn_up8_scores_bwd_workspace_bytes(B, h, w, C, &need) == PCNN_OK, "up8_scores_bwd: bad shape");
    PCNN_REQUIRE(workspace_bytes >= need, "up8_scores_bwd: workspace too small (%zu < %zu)", workspace_bytes, need);
    return up8_bwd_launch(kTargetNone, prob, score, gt, cls_loss_out, upstream_cls, threshold, nullptr, nullptr, nullptr, nullptr, nullptr,
                          nullptr, 0.f, 0.f, 1.f, B, h, w, C, Cs, 0, d_sc_bf16, nullptr, dbias, workspace, stream);
}

extern "C" int pcnn_pose_chain_bwd(const float* bottom_diff, const float* poses_tanh, const float* poses_weight, int N, int D, float upstream,
                                   void* dpre_f16, int ld, void* stream)
{
    PCNN_REQUIRE(bottom_diff && poses_tanh && poses_weight && dpre_f16 && N >= 1 && D >= 1 && ld >= D, "pose_chain_bwd: bad arguments");
    k_pose_chain_bwd<<<(N + 7) / 8, 256, 0, (cudaStream_t)stream>>>(bottom_diff, poses_tanh, poses_weight, N, D, upstream, (__half*)dpre_f16, ld);
    return check_launch("pose_chain_bwd");
}

// accum = mu * accum + (gscale * grad + wd * w); w -= lr * accum; copy16 (optional) = the refreshed tensor-core copy, kind 0 = bf16, 1 = fp16
extern "C" int pcnn_sgd_momentum(float* w, float* accum, const float* grad, size_t n, float lr, float mu, float wd, float gscale, void* copy16,
                                 int kind, void* stream)
{
    PCNN_REQUIRE(w && accum && grad, "sgd_momentum: NULL tensor pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (kind == 1) k_sgd_momentum<__half><<<ew_blocks(n), 256, 0, st>>>(w, accum, grad, n, lr, mu, wd, gscale, (__half*)copy16);
    else k_sgd_momentum<__nv_bfloat16><<<ew_blocks(n), 256, 0, st>>>(w, accum, grad, n, lr, mu, wd, gscale, (__nv_bfloat16*)copy16);
    return check_launch("sgd_momentum");
}

extern "C" int pcnn_transpose16(const void* in, int rows, int cols, void* out, void* stream)
{
    PCNN_REQUIRE(in && out && rows >= 1 && cols >= 1, "transpose16: bad arguments");
    dim3 grid((cols + 63) / 64, (rows + 63) / 64);
    k_transpose16<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)in, rows, cols, (uint16_t*)out);
    return check_launch("transpose16");
}

extern "C" int pcnn_half_to_float(const void* src_f16, size_t n, float scale, float* dst, void* stream)
{
    PCNN_REQUIRE(src_f16 && dst, "half_to_float: NULL tensor pointer");
    k_half_to_float<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>((const __half*)src_f16, n, scale, dst);
    return check_launch("half_to_float");
}
