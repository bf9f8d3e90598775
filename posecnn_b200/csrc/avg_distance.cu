// avg_distance.cu — Averagedistance (ADD / ADD-S pose loss) for sm_90a.
//
// Behavioural spec: lib/average_distance_loss/average_distance_loss_op_gpu.cu.cc:34-252
// (per (roi, point) thread, 54-float rotation scratch + [N,P,4C] diff scratch in global
// memory, two reduction kernels, thrust::reduce and a host round trip).
// Here: one CTA per ROI row, rotations in registers, the gt-rotated model points of a
// symmetric class staged once in shared memory for the closest-point search, block tree
// reductions in a fixed order (deterministic), the batch loss reduced by the last CTA to
// finish — one launch, no scratch tensors, no host synchronisation.
#include <float.h>

#include "common.cuh"

namespace pcnn {

constexpr int kAdThreads = 256;

__device__ __forceinline__ void quat_to_rot(float s, float u, float v, float w, float* R)
{
    // un-normalised quaternion formula of .cu.cc:63-71
    R[0] = s * s + u * u - v * v - w * w; R[1] = 2 * (u * v - s * w); R[2] = 2 * (u * w + s * v);
    R[3] = 2 * (u * v + s * w); R[4] = s * s - u * u + v * v - w * w; R[5] = 2 * (v * w - s * u);
    R[6] = 2 * (u * w - s * v); R[7] = 2 * (v * w + s * u); R[8] = s * s - u * u - v * v + w * w;
}

__global__ void __launch_bounds__(kAdThreads)
k_average_distance(const float* __restrict__ pred, const float* __restrict__ target, const float* __restrict__ weight,
                   const float* __restrict__ point, const float* __restrict__ symmetry, int N, int C, int P, float margin,
                   float* __restrict__ loss, float* __restrict__ bottom_diff, float* __restrict__ roi_loss,
                   unsigned* __restrict__ done_ctr)
{
    extern __shared__ float4 sh4[];     // [P] gt-rotated points (symmetric classes only), one 16-byte load each
    __shared__ float s_red[5][kAdThreads];
    __shared__ int s_cls;
    __shared__ bool s_last;
    const int n = blockIdx.x, t = threadIdx.x;
    const int row = 4 * C;
    // zero this row of bottom_diff (the op output is dense [N,4C])
    for (int i = t; i < row; i += kAdThreads) bottom_diff[(size_t)n * row + i] = 0.f;
    if (t == 0) {
        int cls = -1;
        for (int i = 0; i < C; i++)
            if (weight[(size_t)n * row + 4 * i] > 0.f) { cls = i; break; }  // .cu.cc:47-52
        s_cls = cls;
    }
    __syncthreads();
    const int cls = s_cls;
    float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};  // loss, d/ds, d/du, d/dv, d/dw
    if (cls >= 0) {
        const float* tq = target + (size_t)n * row + 4 * cls;
        const float* pq = pred + (size_t)n * row + 4 * cls;
        float Rg[9], Ru[9];
        quat_to_rot(tq[0], tq[1], tq[2], tq[3], Rg);
        const float s = pq[0], u = pq[1], v = pq[2], w = pq[3];
        quat_to_rot(s, u, v, w, Ru);
        const float* pts = point + (size_t)cls * P * 3;
        const bool sym = symmetry[cls] > 0.f;
        if (sym) {
            for (int i = t; i < P; i += kAdThreads) {
                float q0 = pts[3 * i], q1 = pts[3 * i + 1], q2 = pts[3 * i + 2];
                sh4[i] = make_float4(Rg[0] * q0 + Rg[1] * q1 + Rg[2] * q2, Rg[3] * q0 + Rg[4] * q1 + Rg[5] * q2,
                                     Rg[6] * q0 + Rg[7] * q1 + Rg[8] * q2, 0.f);
            }
            __syncthreads();
        }
        const float inv_np = 1.f / ((float)N * (float)P);
        for (int p = t; p < P; p += kAdThreads) {
            const float q0 = pts[3 * p], q1 = pts[3 * p + 1], q2 = pts[3 * p + 2];
            const float x1 = Ru[0] * q0 + Ru[1] * q1 + Ru[2] * q2;
            const float y1 = Ru[3] * q0 + Ru[4] * q1 + Ru[5] * q2;
            const float z1 = Ru[6] * q0 + Ru[7] * q1 + Ru[8] * q2;
            float x2, y2, z2;
            if (sym) {
                float dmin = FLT_MAX;
                int jmin = 0;
#pragma unroll 8
                for (int i = 0; i < P; i++) {  // first minimum wins, .cu.cc:152-169
                    const float4 g4 = sh4[i];
                    float ex = x1 - g4.x, ey = y1 - g4.y, ez = z1 - g4.z;
                    float dd = ex * ex + ey * ey + ez * ez;
                    if (dd < dmin) { dmin = dd; jmin = i; }
                }
                const float4 gm = sh4[jmin];
                x2 = gm.x; y2 = gm.y; z2 = gm.z;
            } else {
                x2 = Rg[0] * q0 + Rg[1] * q1 + Rg[2] * q2;
                y2 = Rg[3] * q0 + Rg[4] * q1 + Rg[5] * q2;
                z2 = Rg[6] * q0 + Rg[7] * q1 + Rg[8] * q2;
            }
            const float e0 = x1 - x2, e1 = y1 - y2, e2 = z1 - z2;
            const float dist = e0 * e0 + e1 * e1 + e2 * e2;
            if (dist < margin) continue;  // hinge, .cu.cc:177-178
            acc[0] += (dist - margin) * 0.5f * inv_np;
            // d(Ru x)/dq, the four derivative matrices of .cu.cc:96-139 contracted with e and x
            const float a0 = e0 * q0, a1 = e0 * q1, a2 = e0 * q2;
            const float b0 = e1 * q0, b1 = e1 * q1, b2 = e1 * q2;
            const float c0 = e2 * q0, c1 = e2 * q1, c2 = e2 * q2;
            const float gs = 2.f * (a0 * s - a1 * w + a2 * v + b0 * w + b1 * s - b2 * u - c0 * v + c1 * u + c2 * s);
            const float gu = 2.f * (a0 * u + a1 * v + a2 * w + b0 * v - b1 * u - b2 * s + c0 * w + c1 * s - c2 * u);
            const float gv = 2.f * (-a0 * v + a1 * u + a2 * s + b0 * u + b1 * v + b2 * w - c0 * s + c1 * w - c2 * v);
            const float gw = 2.f * (-a0 * w - a1 * s + a2 * u + b0 * s - b1 * w + b2 * v + c0 * u + c1 * v + c2 * w);
            acc[1] += gs * inv_np; acc[2] += gu * inv_np; acc[3] += gv * inv_np; acc[4] += gw * inv_np;
        }
    }
#pragma unroll
    for (int k = 0; k < 5; k++) s_red[k][t] = acc[k];
    __syncthreads();
    for (int o = kAdThreads / 2; o > 0; o >>= 1) {
        if (t < o) {
#pragma unroll
            for (int k = 0; k < 5; k++) s_red[k][t] += s_red[k][t + o];
        }
        __syncthreads();
    }
    if (t == 0) {
        if (cls >= 0)
            for (int k = 0; k < 4; k++) bottom_diff[(size_t)n * row + 4 * cls + k] = s_red[1 + k][0];
        roi_loss[n] = s_red[0][0];
        __threadfence();
        unsigned prev = atomicAdd(done_ctr, 1u);
        s_last = (prev == (unsigned)N - 1);
    }
    __syncthreads();
    if (s_last) {
        // batch loss: fixed-order tree over the per-ROI losses (thrust::reduce + host copy in the reference)
        __threadfence();
        float v = 0.f;
        for (int i = t; i < N; i += kAdThreads) v += roi_loss[i];
        s_red[0][t] = v;
        __syncthreads();
        for (int o = kAdThreads / 2; o > 0; o >>= 1) {
            if (t < o) s_red[0][t] += s_red[0][t + o];
            __syncthreads();
        }
        if (t == 0) { loss[0] = s_red[0][0]; *done_ctr = 0; }
    }
}

__global__ void k_scale(const float* __restrict__ top_diff, const float* __restrict__ bottom_diff, size_t n,
                        float* __restrict__ out)
{
    const float g = top_diff[0];  // .cu.cc:346-354
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = g * bottom_diff[i];
}

}  // namespace pcnn

using namespace pcnn;

extern "C" int pcnn_average_distance_workspace_bytes(int N, size_t* bytes)
{
    PCNN_REQUIRE(N >= 0 && bytes, "average_distance: bad arguments");
    *bytes = 256 + sizeof(float) * (size_t)(N > 0 ? N : 1);
    return PCNN_OK;
}

extern "C" int pcnn_average_distance_fwd(const float* prediction, const float* target, const float* weight,
                                            const float* point, const float* symmetry, int N, int C, int P, float margin,
                                            float* loss, float* bottom_diff, void* workspace, size_t workspace_bytes,
                                            void* stream)
{
    PCNN_REQUIRE(margin >= 0, "Need margin >= 0, got %f", margin);  // average_distance_loss_op.cc:66-68
    PCNN_REQUIRE(prediction && target && weight && point && symmetry && loss && bottom_diff && workspace,
                 "average_distance: NULL tensor pointer");
    PCNN_REQUIRE(N >= 0 && C >= 1 && P >= 1, "average_distance: bad shape");
    size_t need = 0;
    pcnn_average_distance_workspace_bytes(N, &need);
    if (workspace_bytes < need) {
        set_error("average_distance: workspace too small (%zu < %zu)", workspace_bytes, need);
        return PCNN_E_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(workspace, 0, 256, st);  // completion counter
    cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (N == 0) return PCNN_OK;
    size_t smem = sizeof(float4) * (size_t)P;
    PCNN_REQUIRE(smem <= 200 * 1024, "average_distance: P = %d model points exceed the shared-memory staging", P);
    PCNN_SMEM_OPTIN(k_average_distance, 200 * 1024, "average_distance");
    k_average_distance<<<N, kAdThreads, smem, st>>>(prediction, target, weight, point, symmetry, N, C, P, margin, loss,
                                                    bottom_diff, (float*)((char*)workspace + 256), (unsigned*)workspace);
    return check_launch("average_distance_fwd");
}

extern "C" int pcnn_average_distance_bwd(const float* top_diff, const float* bottom_diff, int N, int channels,
                                         float* output, void* stream)
{
    PCNN_REQUIRE(top_diff && bottom_diff && output, "average_distance_grad: NULL tensor pointer");
    size_t n = (size_t)N * channels;
    if (n == 0) return PCNN_OK;
    k_scale<<<(int)((n + 255) / 256 > 1184 ? 1184 : (n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(top_diff, bottom_diff,
                                                                                                     n, output);
    return check_launch("average_distance_bwd");
}
