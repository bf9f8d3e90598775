// heads_common.cuh — the bilinear x8 transposed convolution of the FCN heads, shared by k_up8_heads (heads.cu, dense
// vertex_pred) and the Hough sampler (hough_vote.cu, k_emit: vertex values of the sampled pixels only).  Both go
// through the SAME operation sequence, so a value computed on demand is bit-identical to the dense tensor's.
#pragma once
#include "common.cuh"

namespace pcnn {

// make_deconv_filter (network.py:141-157): f = ceil(k/2), c = (2f - 1 - f%2) / (2f), W[x] = 1 - |x/f - c|
__host__ __device__ inline float deconv_w(int x, int k)
{
    // k = 16: f = 8, c = 15/16; k = 4: f = 2, c = 3/4 (exact in binary floating point)
    if (k == 16) return 1.f - fabsf((float)x * 0.125f - 0.9375f);
    if (k == 4) return 1.f - fabsf((float)x * 0.5f - 0.75f);
    int f = (k + 1) / 2;
    float c = (2.f * f - 1.f - (float)(f % 2)) / (2.f * f);
    return 1.f - fabsf((float)x / (float)f - c);
}

// vertical blend of the two contributing low-resolution rows (what k_up8_heads stages in shared memory)
__device__ __forceinline__ float up8_vblend(float wy0, float a, float wy1, float b) { return fmaf(wy1, b, __fmul_rn(wy0, a)); }
// horizontal blend of two staged values + bias (one output value)
__device__ __forceinline__ float up8_hblend(float wa, float a, float wb, float b, float bias)
{
    return __fadd_rn(fmaf(wb, b, __fmul_rn(wa, a)), bias);
}

// One value of up8(lowres)[n, y, x, ch] + bias: conv2d_transpose 16x16 / stride 8, SAME (pad 4):
// out[o] = sum_i in[i] * W[o - 8 i + 4].  lr = [B, h, w, No] f32.
__device__ __forceinline__ float up8_value(const float* __restrict__ lr, int n, int h, int w, int No, int ch, int y, int x,
                                           float bias)
{
    const int my = y >> 3, ty = y & 7;
    const int iy0 = ty < 4 ? my - 1 : my, iy1 = iy0 + 1;
    const float wy0 = (iy0 >= 0 && iy0 < h) ? deconv_w(y - 8 * iy0 + 4, 16) : 0.f;
    const float wy1 = (iy1 >= 0 && iy1 < h) ? deconv_w(y - 8 * iy1 + 4, 16) : 0.f;
    const float* r0 = lr + ((size_t)n * h + min(max(iy0, 0), h - 1)) * w * No + ch;
    const float* r1 = lr + ((size_t)n * h + min(max(iy1, 0), h - 1)) * w * No + ch;
    const int mx = x >> 3, tx = x & 7;
    const int ia = tx < 4 ? mx - 1 : mx, ib = ia + 1;
    const float wa = deconv_w(tx < 4 ? tx + 12 : tx + 4, 16), wb = deconv_w(tx < 4 ? tx + 4 : tx - 4, 16);
    const float va = (ia >= 0 && ia < w) ? up8_vblend(wy0, __ldg(r0 + (size_t)ia * No), wy1, __ldg(r1 + (size_t)ia * No)) : 0.f;
    const float vb = (ib >= 0 && ib < w) ? up8_vblend(wy0, __ldg(r0 + (size_t)ib * No), wy1, __ldg(r1 + (size_t)ib * No)) : 0.f;
    return up8_hblend(wa, va, wb, vb, bias);
}

// _scale_vertmap (minibatch.py:605-616), the VERTEX_REG_3D target of one class, shared by the fused loss (train_targets.cu) and the
// up-sampling adjoint (train_bwd.cu).  The reference works in float32 (extents and vertmap are float32 arrays), so vmin = -e / 2,
// vmax = e / 2, a = 1 / (vmax - vmin), b = -1 * vmin / (vmax - vmin) are float32 operations (a = b = 0 where vmax - vmin <= 0), and
// the target of an object coordinate v is a * v rounded, then + b rounded: no contraction into an FMA.  ab = (a_0, b_0, a_1, ..).
__device__ __forceinline__ void coord_scale(const float* ext /*[3]*/, float ab[6])
{
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float e = ext[k];
        const float vmin = -e / 2.f, vmax = e / 2.f, span = vmax - vmin;
        const bool ok = span > 0.f;
        ab[2 * k] = ok ? 1.f / span : 0.f;
        ab[2 * k + 1] = ok ? (-1.f * vmin) / span : 0.f;
    }
}

__device__ __forceinline__ float coord_target(float a, float b, float v) { return __fadd_rn(__fmul_rn(a, v), b); }

}  // namespace pcnn
