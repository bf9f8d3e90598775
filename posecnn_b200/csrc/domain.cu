// domain.cu — the domain-adaptation branch of vgg16_convs (lib/networks/vgg16_convs.py:202-212; loss lib/fcn/train.py:508-513):
//   pool_score -> gradient_reversal(lambda) -> fc9 (25088 -> 256, ReLU) -> domain_score = fc(2) -> softmax -> argmax
// domain_score is built with Network.fc's default relu=True (network.py:393,420), so the two logits pass through a ReLU.
// fc9's three GEMMs run on the fully connected kernels (csrc/fc_tc.cu, csrc/wgrad_tc.cu); this file holds the pieces around them:
//   k_domain_tail   ONE CTA: per row, the 256 -> 2 layer, its ReLU, softmax and arg-max; with labels also the cross entropy and
//                   its gradient back through the ReLU, the 256 -> 2 layer and fc9's ReLU (mask = fc9's stored fp16 output > 0).
//                   Warp w takes rows w, w + 16, ...; every per-warp partial (loss, dW10, db10, db9) is summed over the warps in
//                   index order through shared memory: a fixed order, no atomics, two launches are bit-identical.
//   k_domain_merge  dpool = s_a * a + s_b * b from the pose head's and the domain branch's fp16 input gradients of pool_score;
//                   s_b = -lambda / S_d is the gradient reversal.  s_a * a is one fp32 multiply, as k_half_to_float forms it.
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"

namespace pcnn {
namespace domain {

constexpr int kHid = 256;                  // fc9 units
constexpr int kWarps = 16;
constexpr int kThreads = kWarps * 32;
constexpr int kPer = kHid / 32;            // hidden units per lane: k = kPer * lane + j

// the fixed-order sum over warps of one [kHid] partial held as v[kPer] by every lane -> dst[kHid]
__device__ __forceinline__ void reduce_warps(const float (&v)[kPer], float (*red)[kHid], int warp, int k0, float* __restrict__ dst)
{
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kPer; j++) red[warp][k0 + j] = v[j];
    __syncthreads();
    if (threadIdx.x < kHid) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; w++) s += red[w][threadIdx.x];
        dst[threadIdx.x] = s;
    }
}

__global__ void __launch_bounds__(kThreads, 1)
k_domain_tail(const __half* __restrict__ h9, int rows, int ld, const float* __restrict__ w10 /*[2][256]*/, const float* __restrict__ b10,
              const int32_t* __restrict__ label_domain, float loss_scale, float grad_scale, float* __restrict__ score,
              float* __restrict__ prob, int32_t* __restrict__ label, float* __restrict__ loss, float* __restrict__ amax,
              float* __restrict__ dw10, float* __restrict__ db10, float* __restrict__ db9, __half* __restrict__ dpre9)
{
    __shared__ float red[kWarps][kHid];
    __shared__ float red_s[kWarps][4];     // loss, max |d fc9 pre-activation|, db10[0], db10[1]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k0 = kPer * lane;
    const bool train = label_domain != nullptr;
    float w0[kPer], w1[kPer], g0[kPer], g1[kPer], g9[kPer];
#pragma unroll
    for (int j = 0; j < kPer; j++) {
        w0[j] = __ldg(w10 + k0 + j);
        w1[j] = __ldg(w10 + kHid + k0 + j);
        g0[j] = g1[j] = g9[j] = 0.f;
    }
    const float bias0 = __ldg(b10), bias1 = __ldg(b10 + 1);
    float sl = 0.f, sb0 = 0.f, sb1 = 0.f, mx = 0.f;
    for (int r = warp; r < rows; r += kWarps) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(h9 + (size_t)r * ld + k0));
        const __half2* hp = reinterpret_cast<const __half2*>(&raw);
        float h[kPer];
#pragma unroll
        for (int j = 0; j < kPer / 2; j++) {
            const float2 f = __half22float2(hp[j]);
            h[2 * j] = f.x;
            h[2 * j + 1] = f.y;
        }
        float p0 = 0.f, p1 = 0.f;
#pragma unroll
        for (int j = 0; j < kPer; j++) { p0 = fmaf(h[j], w0[j], p0); p1 = fmaf(h[j], w1[j], p1); }
        // butterfly: a + b == b + a, so every lane ends with the same sums
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { p0 += __shfl_xor_sync(0xffffffffu, p0, o); p1 += __shfl_xor_sync(0xffffffffu, p1, o); }
        const float z0 = fmaxf(p0 + bias0, 0.f), z1 = fmaxf(p1 + bias1, 0.f);
        const float m = fmaxf(z0, z1);
        const float e0 = expf(z0 - m), e1 = expf(z1 - m), s = e0 + e1;
        const float q0 = e0 / s, q1 = e1 / s;
        if (lane == 0) {
            score[2 * r] = z0; score[2 * r + 1] = z1;
            prob[2 * r] = q0; prob[2 * r + 1] = q1;
            label[r] = z1 > z0 ? 1 : 0;                    // first maximum on ties
        }
        if (!train) continue;
        const int lab = label_domain[r] == 1 ? 1 : 0;
        sl += (m + logf(s)) - (lab ? z1 : z0);             // sparse softmax cross entropy of the row
        // d loss / d pre-activation of domain_score: (softmax - onehot) where the ReLU passed (TF ReluGrad: output > 0).
        // q[label] - 1 is formed as -q[other] (q0 + q1 = 1): no cancellation when the softmax saturates
        const float gz0 = z0 > 0.f ? loss_scale * (lab == 0 ? -q1 : q0) : 0.f;
        const float gz1 = z1 > 0.f ? loss_scale * (lab == 1 ? -q0 : q1) : 0.f;
        sb0 += gz0;
        sb1 += gz1;
        float d[kPer];
#pragma unroll
        for (int j = 0; j < kPer; j++) {
            g0[j] = fmaf(gz0, h[j], g0[j]);
            g1[j] = fmaf(gz1, h[j], g1[j]);
            d[j] = h[j] > 0.f ? fmaf(gz1, w1[j], gz0 * w0[j]) : 0.f;      // through fc9's ReLU
            g9[j] += d[j];
            mx = fmaxf(mx, fabsf(d[j]));
        }
        uint4 pk;
        __half2* po = reinterpret_cast<__half2*>(&pk);
#pragma unroll
        for (int j = 0; j < kPer / 2; j++) po[j] = __floats2half2_rn(sat_f16(grad_scale * d[2 * j]), sat_f16(grad_scale * d[2 * j + 1]));
        *reinterpret_cast<uint4*>(dpre9 + (size_t)r * ld + k0) = pk;
        for (int c = kHid + lane; c < ld; c += 32) dpre9[(size_t)r * ld + c] = __float2half_rn(0.f);
    }
    if (!train) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) { red_s[warp][0] = sl; red_s[warp][1] = mx; red_s[warp][2] = sb0; red_s[warp][3] = sb1; }
    reduce_warps(g0, red, warp, k0, dw10);
    reduce_warps(g1, red, warp, k0, dw10 + kHid);
    reduce_warps(g9, red, warp, k0, db9);
    if (threadIdx.x == 0) {
        float l = 0.f, a = 0.f, c0 = 0.f, c1 = 0.f;
        for (int w = 0; w < kWarps; w++) { l += red_s[w][0]; a = fmaxf(a, red_s[w][1]); c0 += red_s[w][2]; c1 += red_s[w][3]; }
        loss[0] = loss_scale * l;
        amax[0] = a;
        db10[0] = c0;
        db10[1] = c1;
    }
}

// dst[i] = s_a * a[i] + s_b * b[i], eight elements per iteration; both products rounded before the add (no fused multiply-add)
__global__ void __launch_bounds__(256)
k_domain_merge(const __half* __restrict__ a, float sa, const __half* __restrict__ b, float sb, size_t n8, float* __restrict__ dst)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 va = __ldg(reinterpret_cast<const uint4*>(a) + i), vb = __ldg(reinterpret_cast<const uint4*>(b) + i);
        const __half2* pa = reinterpret_cast<const __half2*>(&va);
        const __half2* pb = reinterpret_cast<const __half2*>(&vb);
        float o[8];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const float2 fa = __half22float2(pa[j]), fb = __half22float2(pb[j]);
            o[2 * j] = __fadd_rn(__fmul_rn(sa, fa.x), __fmul_rn(sb, fb.x));
            o[2 * j + 1] = __fadd_rn(__fmul_rn(sa, fa.y), __fmul_rn(sb, fb.y));
        }
        float4* d = reinterpret_cast<float4*>(dst) + 2 * i;
        st_stream_f4(d, make_float4(o[0], o[1], o[2], o[3]));
        st_stream_f4(d + 1, make_float4(o[4], o[5], o[6], o[7]));
    }
}

}  // namespace domain
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::domain;

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" int pcnn_domain_tail(const void* fc9_f16, int rows, int ld, const float* w10, const float* b10, const int32_t* label_domain,
                                float loss_scale, float grad_scale, float* domain_score, float* domain_prob, int32_t* domain_label,
                                float* loss, float* amax, float* dw10, float* db10, float* db9, void* dpre9_f16, void* stream)
{
    PCNN_REQUIRE(fc9_f16 && w10 && b10 && domain_score && domain_prob && domain_label, "domain_tail: NULL tensor pointer");
    PCNN_REQUIRE(!label_domain || (loss && amax && dw10 && db10 && db9 && dpre9_f16), "domain_tail: NULL gradient pointer with labels given");
    PCNN_REQUIRE(rows >= 1 && rows <= PCNN_HOUGH_MAX_ROWS, "domain_tail: rows must be in [1, %d] (got %d)", PCNN_HOUGH_MAX_ROWS, rows);
    PCNN_REQUIRE(ld >= kHid && ld % 8 == 0, "domain_tail: ld must be a multiple of 8 and >= %d (got %d)", kHid, ld);
    PCNN_REQUIRE(aligned16(fc9_f16) && (!label_domain || aligned16(dpre9_f16)), "domain_tail: fp16 tensors must be 16-byte aligned");
    PCNN_REQUIRE(!label_domain || grad_scale > 0.f, "domain_tail: grad_scale must be positive");
    k_domain_tail<<<1, kThreads, 0, (cudaStream_t)stream>>>((const __half*)fc9_f16, rows, ld, w10, b10, label_domain, loss_scale, grad_scale,
                                                           domain_score, domain_prob, domain_label, loss, amax, dw10, db10, db9,
                                                           (__half*)dpre9_f16);
    return check_launch("domain_tail");
}

extern "C" int pcnn_domain_grad_merge(const void* a_f16, float scale_a, const void* b_f16, float scale_b, size_t n, float* dst, void* stream)
{
    PCNN_REQUIRE(a_f16 && b_f16 && dst, "domain_grad_merge: NULL tensor pointer");
    PCNN_REQUIRE(n >= 8 && n % 8 == 0, "domain_grad_merge: n must be a positive multiple of 8 (got %zu)", n);
    PCNN_REQUIRE(aligned16(a_f16) && aligned16(b_f16) && aligned16(dst), "domain_grad_merge: tensors must be 16-byte aligned");
    const size_t n8 = n / 8;
    const int blocks = (int)std::min<size_t>((n8 + 255) / 256, (size_t)kNumSMs * 8);
    k_domain_merge<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)a_f16, scale_a, (const __half*)b_f16, scale_b, n8, dst);
    return check_launch("domain_grad_merge");
}
