// train_targets.cu — training-side target generation and the training step's fused losses (SURVEY.md §8(f) rank 3).
//
//   pcnn_vertex_targets_fwd            lib/gt_synthesize_layer/minibatch.py:543-602 (_generate_vertex_targets, the
//                                      single-instance branch :578-599): per labelled pixel of a present class
//                                      (dx, dy) / (|(dx, dy)| + 1e-10) toward the projected centre and log z; weights = W_INSIDE
//   pcnn_vertex_targets_3d_fwd         the VERTEX_REG_3D branch of _generate_vertex_targets (minibatch.py:595-600, _scale_vertmap
//                                      :605-616): the pixel's object coordinate scaled into [0, 1] by its class's extents
//   pcnn_loss_cls_hard_raw_fwd         lib/fcn/train.py:455-465 (loss_cross_entropy_single_frame) on log_softmax(score) over the
//                                      Hardlabel selection (hard_label_op_gpu.cu.cc:16-29), neither tensor materialised
//   pcnn_vertex_loss_fwd               lib/fcn/train.py:564-573 (smooth_l1_loss_vertex) on the targets of either branch, vertex
//                                      values from the 1/8-resolution head tensor, targets / weights never materialised
// Losses: fixed 592-CTA grid, per-CTA partial sums in double, last CTA to finish reduces them in index order
// (run-to-run deterministic).  Their gradients are the up-sampling adjoint's (train_bwd.cu).
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "heads_common.cuh"
#include "pose_common.cuh"

namespace pcnn {

constexpr int kLossBlocks = kNumSMs * 4;
constexpr int kLossThreads = 256;

// ---------------------------------------------------------------------------------------------
// deterministic two-value reduction: per-CTA partials, last CTA sums them in index order
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void block_reduce2(double& a, double& b, double* sh /*[2 * warps]*/)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane == 0) { sh[2 * w] = a; sh[2 * w + 1] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double sa = 0, sb = 0;
        for (int k = 0; k < nw; k++) { sa += sh[2 * k]; sb += sh[2 * k + 1]; }
        a = sa; b = sb;
    }
}

__device__ __forceinline__ bool finish_partials(double a, double b, double* partial /*[2 * grid]*/, unsigned* ticket, double& ta, double& tb)
{
    __shared__ bool last;
    if (threadIdx.x == 0) {
        partial[2 * blockIdx.x] = a; partial[2 * blockIdx.x + 1] = b;
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return false;
    if (threadIdx.x == 0) {
        __threadfence();
        const volatile double* vp = partial;
        double sa = 0, sb = 0;
        for (unsigned k = 0; k < gridDim.x; k++) { sa += vp[2 * k]; sb += vp[2 * k + 1]; }
        ta = sa; tb = sb;
        *ticket = 0;                                       // ready for the next launch
    }
    return threadIdx.x == 0;
}

// cross entropy over the pixels Hardlabel selects (gt != -1 and (gt > 0 or prob[gt] < threshold)) from the RAW scores (the `score`
// layer output): log-softmax of the labelled class computed per selected pixel (network.py:491-506: x - max - log sum exp(x - max)),
// so neither the [B,H,W,C] log-probability tensor nor the mask is materialised
__global__ void __launch_bounds__(kLossThreads)
k_loss_cls_hard_raw(const float* __restrict__ score_raw, const float* __restrict__ prob, const int* __restrict__ gt, unsigned npix, int C,
                    float threshold, double* __restrict__ partial, unsigned* __restrict__ ticket, float* __restrict__ out /*[2]: loss, count*/)
{
    __shared__ double sh[2 * kLossThreads / 32];
    double s = 0, n = 0;
    for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
        const int g = __ldg(gt + p);
        if (g < 0 || g >= C) continue;                     // -1 = ignore (hard_label_op_gpu.cu.cc:24); out-of-range labels ignored
        if (g > 0 || __ldg(prob + (size_t)p * C + g) < threshold) {
            const float* sp = score_raw + (size_t)p * C;
            float m = __ldg(sp);
            for (int c = 1; c < C; c++) m = fmaxf(m, __ldg(sp + c));
            float se = 0.f;
            for (int c = 0; c < C; c++) se += expf(__ldg(sp + c) - m);
            s -= (double)(__ldg(sp + g) - m - logf(se));
            n += 1.0;
        }
    }
    block_reduce2(s, n, sh);
    double ts, tn;
    if (finish_partials(s, n, partial, ticket, ts, tn)) {
        out[0] = (float)(ts / (tn + 1e-10));
        out[1] = (float)tn;
    }
}

// smooth L1 on a weighted difference (train.py:564-573)
__device__ __forceinline__ float sl1_term(float pred, float targ, float wgt, float sigma2)
{
    const float diff = wgt * (pred - targ);
    const float ad = fabsf(diff);
    return ad < 1.f / sigma2 ? diff * diff * (sigma2 * 0.5f) : ad - 0.5f / sigma2;
}

// ---------------------------------------------------------------------------------------------
// vertex targets, and the fused vertex loss: smooth_l1_loss_vertex(vertex_pred, targets(label, ..), weights(label, ..)) without
// the two [B,H,W,3C] target / weight tensors (5.2 GB at batch 32): only the three channels of a labelled pixel's own
// class carry weight, so the loss forms three vertex values per foreground pixel.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool pixel_targets(const int* __restrict__ label, const float* __restrict__ centers, unsigned pix, int HW,
                                              int W, int C, int& cls, float t[3])
{
    const int l = __ldg(label + pix);
    if (l <= 0 || l >= C) return false;
    const int b = pix / HW, p = pix - b * HW;
    const float* cen = centers + ((size_t)b * C + l) * 3;
    const float z = cen[2];
    if (!(z > 0.f)) return false;
    const double dx = (double)cen[0] - (double)(p % W), dy = (double)cen[1] - (double)(p / W);
    const double nrm = sqrt(dx * dx + dy * dy) + 1e-10;
    t[0] = (float)(dx / nrm); t[1] = (float)(dy / nrm); t[2] = (float)log((double)z);
    cls = l;
    return true;
}

// VERTEX_REG_3D target (minibatch.py:595-600 with _scale_vertmap, :605-616; coord_scale / coord_target: heads_common.cuh): the pixel's
// object coordinate vertmap [.., 3] scaled into [0, 1] by its class's extents.  Weighted pixels are those of pixel_targets: label l in
// 1..C-1 with a listed centre (centers[b, l, 2] > 0), so `centers` stays the presence table.
__device__ __forceinline__ bool pixel_targets_3d(const int* __restrict__ label, const float* __restrict__ vertmap, const float* __restrict__ centers,
                                                 const float* __restrict__ extents, unsigned pix, int HW, int C, int& cls, float t[3])
{
    const int l = __ldg(label + pix);
    if (l <= 0 || l >= C) return false;
    const int b = pix / HW;
    if (!(centers[((size_t)b * C + l) * 3 + 2] > 0.f)) return false;
    float ab[6];
    coord_scale(extents + 3 * l, ab);
#pragma unroll
    for (int k = 0; k < 3; k++) t[k] = coord_target(ab[2 * k], ab[2 * k + 1], __ldg(vertmap + (size_t)pix * 3 + k));
    cls = l;
    return true;
}

// the target of either mode: 2-D centre direction + log z (kCoord = false) or the scaled object coordinate (kCoord = true)
template <bool kCoord>
__device__ __forceinline__ bool vertex_target(const int* __restrict__ label, const float* __restrict__ centers, const float* __restrict__ vertmap,
                                              const float* __restrict__ extents, unsigned pix, int HW, int W, int C, int& cls, float t[3])
{
    if constexpr (kCoord) return pixel_targets_3d(label, vertmap, centers, extents, pix, HW, C, cls, t);
    else return pixel_targets(label, centers, pix, HW, W, C, cls, t);
}

// materialised targets / weights (drop-in for the data layer's blobs): the tensors are >97 % zeros, so they are
// cleared with two memset nodes and only the three channels of each labelled pixel's own class are written
__global__ void __launch_bounds__(256)
k_vertex_targets_sparse(const int* __restrict__ label, const float* __restrict__ centers, unsigned npix, int HW, int W, int C, float w_inside,
                        float* __restrict__ targets, float* __restrict__ weights)
{
    for (unsigned pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
        int cls;
        float t[3];
        if (!pixel_targets(label, centers, pix, HW, W, C, cls, t)) continue;
        const size_t o = (size_t)pix * 3 * C + 3 * cls;
#pragma unroll
        for (int k = 0; k < 3; k++) { targets[o + k] = t[k]; weights[o + k] = w_inside; }
    }
}

// the same for the VERTEX_REG_3D target (pixel_targets_3d)
__global__ void __launch_bounds__(256)
k_vertex_targets_3d_sparse(const int* __restrict__ label, const float* __restrict__ vertmap, const float* __restrict__ centers,
                           const float* __restrict__ extents, unsigned npix, int HW, int C, float w_inside, float* __restrict__ targets,
                           float* __restrict__ weights)
{
    for (unsigned pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
        int cls;
        float t[3];
        if (!pixel_targets_3d(label, vertmap, centers, extents, pix, HW, C, cls, t)) continue;
        const size_t o = (size_t)pix * 3 * C + 3 * cls;
#pragma unroll
        for (int k = 0; k < 3; k++) { targets[o + k] = t[k]; weights[o + k] = w_inside; }
    }
}

// multi-instance branch of _generate_vertex_targets (minibatch.py:549-573): several instances of one class in an image
// are told apart by an instance-mask image; instance i = (cls, mask id = cls_indexes_old[i] + 1, projected centre, z)
// owns the pixels with mask == id AND label == cls.  The reference loops the instances in order and overwrites, so the
// LAST matching instance wins.  instances [B, I, 5] = (cls, mask_id, cx, cy, z); z <= 0 marks an unused slot.
__global__ void __launch_bounds__(256)
k_vertex_targets_instances(const int* __restrict__ label, const int* __restrict__ mask, const float* __restrict__ inst, unsigned npix,
                           int HW, int W, int C, int I, float w_inside, float* __restrict__ targets, float* __restrict__ weights)
{
    for (unsigned pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
        const int l = __ldg(label + pix);
        if (l <= 0 || l >= C) continue;
        const int m = __ldg(mask + pix);
        const int b = pix / HW, p = pix - b * HW;
        const float* rows = inst + (size_t)b * I * 5;
        int hit = -1;
        for (int i = 0; i < I; i++)
            if (rows[5 * i + 4] > 0.f && (int)rows[5 * i] == l && (int)rows[5 * i + 1] == m) hit = i;
        if (hit < 0) continue;
        const float* r = rows + 5 * hit;
        const double dx = (double)r[2] - (double)(p % W), dy = (double)r[3] - (double)(p / W);
        const double nrm = sqrt(dx * dx + dy * dy) + 1e-10;
        const size_t o = (size_t)pix * 3 * C + 3 * l;
        targets[o] = (float)(dx / nrm); targets[o + 1] = (float)(dy / nrm); targets[o + 2] = (float)log((double)r[4]);
        weights[o] = w_inside; weights[o + 1] = w_inside; weights[o + 2] = w_inside;
    }
}

// ---------------------------------------------------------------------------------------------
// pose blob and meta_data packing of the data layer (minibatch.py:440-451, 474-492):
//   pose_blob rows [image, cls, 0, 0, 0, 0, mat2quat(R) (w, x, y, z), T] for every listed instance, images in order;
//   meta_data[48]: K * im_scale with K[2][2] = 1 in [0:9], its (pseudo-)inverse in [9:18], zeros elsewhere, FLIP_X signs.
// mat2quat_d: pose_common.cuh.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_pack_pose_meta(const float* __restrict__ poses /*[B,I,12]*/, const int* __restrict__ cls /*[B,I], < 0 = unused*/,
                 const float* __restrict__ intr /*[B,9]*/, int B, int I, float im_scale, int flip_x, float* __restrict__ pose_blob /*[B*I,13]*/,
                 int* __restrict__ num_rows, float* __restrict__ meta /*[B,48]*/)
{
    __shared__ int s_off[1025];
    const int t = threadIdx.x, n = B * I;
    if (t == 0) {
        int run = 0;
        for (int k = 0; k < n; k++) { s_off[k] = run; run += cls[k] >= 0 ? 1 : 0; }
        s_off[n] = run;
        *num_rows = run;
    }
    __syncthreads();
    for (int k = t; k < n; k += blockDim.x) {
        float* row = pose_blob + (size_t)k * 13;
        if (k >= s_off[n])
            for (int j = 0; j < 13; j++) row[j] = 0.f;      // rows beyond the count are zero (capacity buffer)
    }
    __syncthreads();
    for (int k = t; k < n; k += blockDim.x) {
        if (cls[k] < 0) continue;
        const float* rt = poses + (size_t)k * 12;
        float* row = pose_blob + (size_t)s_off[k] * 13;
        row[0] = (float)(k / I); row[1] = (float)cls[k];
        row[2] = row[3] = row[4] = row[5] = 0.f;            // box: "fill later" (minibatch.py:447)
        mat2quat_d(rt, row + 6);
        row[10] = rt[3]; row[11] = rt[7]; row[12] = rt[11];
    }
    for (int b = t; b < B; b += blockDim.x) {
        float* m = meta + (size_t)b * 48;
        for (int j = 0; j < 48; j++) m[j] = 0.f;
        double K[9];
        for (int j = 0; j < 9; j++) K[j] = (double)(float)(intr[b * 9 + j]) * (double)im_scale;
        K[8] = 1.0;
        // inverse by cofactors (np.linalg.pinv of the non-singular 3x3; agreement 1e-6 relative after the float32 cast)
        const double c00 = K[4] * K[8] - K[5] * K[7], c01 = K[5] * K[6] - K[3] * K[8], c02 = K[3] * K[7] - K[4] * K[6];
        const double det = K[0] * c00 + K[1] * c01 + K[2] * c02;
        double Ki[9] = {c00 / det, (K[2] * K[7] - K[1] * K[8]) / det, (K[1] * K[5] - K[2] * K[4]) / det,
                        c01 / det, (K[0] * K[8] - K[2] * K[6]) / det, (K[2] * K[3] - K[0] * K[5]) / det,
                        c02 / det, (K[1] * K[6] - K[0] * K[7]) / det, (K[0] * K[4] - K[1] * K[3]) / det};
        for (int j = 0; j < 9; j++) { m[j] = (float)K[j]; m[9 + j] = (float)Ki[j]; }
        if (flip_x) { m[0] = -m[0]; m[9] = -m[9]; m[11] = -m[11]; }   // minibatch.py:488-491
    }
}

// kCoord: the VERTEX_REG_3D target (vertmap + extents, pixel_targets_3d); otherwise the 2-D one (vertmap / extents unused)
template <bool kCoord>
__global__ void __launch_bounds__(kLossThreads)
k_vertex_loss_fused(const float* __restrict__ lowres, const float* __restrict__ bias_v, const int* __restrict__ label,
                    const float* __restrict__ centers, unsigned npix, int HW, int W, int C, float w_inside, float sigma2,
                    double* __restrict__ partial, unsigned* __restrict__ ticket, float* __restrict__ out /*[2]: loss, sum w*/,
                    const float* __restrict__ vertmap, const float* __restrict__ extents)
{
    // the labelled pixels' three vertex values are formed on demand from the 1/8-resolution head tensor with k_up8_heads' own
    // operation sequence (heads_common.cuh) — bit-identical to reading the dense vertex_pred
    __shared__ double sh[2 * kLossThreads / 32];
    double s = 0, sw = 0;
    for (unsigned pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
        int cls;
        float t[3];
        if (!vertex_target<kCoord>(label, centers, vertmap, extents, pix, HW, W, C, cls, t)) continue;
        const int b = pix / HW, pp = pix - b * HW, y = pp / W, x = pp - y * W;
        float v[3];                                        // all three loads in flight before the first term
#pragma unroll
        for (int k = 0; k < 3; k++) v[k] = up8_value(lowres, b, (HW / W) >> 3, W >> 3, 4 * C, C + 3 * cls + k, y, x, __ldg(bias_v + 3 * cls + k));
#pragma unroll
        for (int k = 0; k < 3; k++) s += (double)sl1_term(v[k], t[k], w_inside, sigma2);
        sw += 3.0 * (double)w_inside;
    }
    block_reduce2(s, sw, sh);
    double ts, tw;
    if (finish_partials(s, sw, partial, ticket, ts, tw)) {
        out[0] = (float)(ts / (tw + 1e-10));               // train.py:572
        out[1] = (float)tw;
    }
}

}  // namespace pcnn

using namespace pcnn;

// the vertex head given as the 1/8-resolution head tensor `lowres` [B,H/8,W/8,4C] (channels C.. = vertex) + the vertex_pred bias
// [3C]: no dense vertex_pred tensor is needed anywhere in the training step.  vertmap and extents both NULL: the 2-D target; both
// given: the VERTEX_REG_3D scaled object-coordinate target (pixel_targets_3d)
extern "C" int pcnn_vertex_loss_fwd(const float* lowres, const float* bias_vertex, const int32_t* label, const float* centers,
                                    const float* vertmap, const float* extents, int B, int H, int W, int C, float w_inside, float sigma,
                                    float* loss_out, void* workspace, size_t workspace_bytes, void* stream)
{
    PCNN_REQUIRE(lowres && bias_vertex && label && centers && loss_out && workspace, "vertex_loss: NULL tensor pointer");
    PCNN_REQUIRE(!vertmap == !extents, "vertex_loss: vertmap and extents must both be given (3-D target) or both be NULL (2-D target)");
    PCNN_REQUIRE(sigma > 0.f && B >= 1 && H >= 8 && W >= 8 && H % 8 == 0 && W % 8 == 0 && C >= 1, "vertex_loss: bad arguments");
    PCNN_REQUIRE((unsigned long long)B * H * W < 0xffffffffULL, "vertex_loss: too many pixels");
    size_t need = 0;
    pcnn_train_loss_workspace_bytes(&need);
    PCNN_REQUIRE(workspace_bytes >= need, "vertex_loss: workspace too small (%zu < %zu)", workspace_bytes, need);
    double* partial = (double*)workspace;
    unsigned* ticket = (unsigned*)(partial + 2 * kLossBlocks);
    (vertmap ? k_vertex_loss_fused<true> : k_vertex_loss_fused<false>)<<<kLossBlocks, kLossThreads, 0, (cudaStream_t)stream>>>(
        lowres, bias_vertex, label, centers, (unsigned)B * H * W, H * W, W, C, w_inside, sigma * sigma, partial, ticket, loss_out, vertmap,
        extents);
    return check_launch("vertex_loss");
}

extern "C" int pcnn_train_loss_workspace_bytes(size_t* bytes)
{
    PCNN_REQUIRE(bytes, "train_loss_workspace_bytes: NULL pointer");
    *bytes = sizeof(double) * 2 * kLossBlocks + 16;        // per-CTA partials + ticket (must be zero on first use)
    return PCNN_OK;
}

extern "C" int pcnn_vertex_targets_fwd(const int32_t* label, const float* centers, int B, int H, int W, int C, float w_inside,
                                       float* targets, float* weights, void* stream)
{
    PCNN_REQUIRE(label && centers && targets && weights, "vertex_targets: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 1, "vertex_targets: bad shape");
    PCNN_REQUIRE((unsigned long long)B * H * W < 0xffffffffULL, "vertex_targets: too many pixels");
    const unsigned npix = (unsigned)B * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(targets, 0, sizeof(float) * (size_t)npix * 3 * C, st);
    cudaMemsetAsync(weights, 0, sizeof(float) * (size_t)npix * 3 * C, st);
    k_vertex_targets_sparse<<<kNumSMs * 16, 256, 0, st>>>(label, centers, npix, H * W, W, C, w_inside, targets, weights);
    return check_launch("vertex_targets");
}

extern "C" int pcnn_vertex_targets_3d_fwd(const int32_t* label, const float* vertmap, const float* centers, const float* extents, int B, int H,
                                          int W, int C, float w_inside, float* targets, float* weights, void* stream)
{
    PCNN_REQUIRE(label && vertmap && centers && extents && targets && weights, "vertex_targets_3d: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 1, "vertex_targets_3d: bad shape");
    PCNN_REQUIRE((unsigned long long)B * H * W < 0xffffffffULL, "vertex_targets_3d: too many pixels");
    const unsigned npix = (unsigned)B * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(targets, 0, sizeof(float) * (size_t)npix * 3 * C, st);
    cudaMemsetAsync(weights, 0, sizeof(float) * (size_t)npix * 3 * C, st);
    k_vertex_targets_3d_sparse<<<kNumSMs * 16, 256, 0, st>>>(label, vertmap, centers, extents, npix, H * W, C, w_inside, targets, weights);
    return check_launch("vertex_targets_3d");
}

extern "C" int pcnn_vertex_targets_instances_fwd(const int32_t* label, const int32_t* mask, const float* instances, int B, int H, int W,
                                                 int C, int I, float w_inside, float* targets, float* weights, void* stream)
{
    PCNN_REQUIRE(label && mask && instances && targets && weights, "vertex_targets_instances: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 1 && I >= 1, "vertex_targets_instances: bad shape");
    PCNN_REQUIRE((unsigned long long)B * H * W < 0xffffffffULL, "vertex_targets_instances: too many pixels");
    const unsigned npix = (unsigned)B * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(targets, 0, sizeof(float) * (size_t)npix * 3 * C, st);
    cudaMemsetAsync(weights, 0, sizeof(float) * (size_t)npix * 3 * C, st);
    k_vertex_targets_instances<<<kNumSMs * 16, 256, 0, st>>>(label, mask, instances, npix, H * W, W, C, I, w_inside, targets, weights);
    return check_launch("vertex_targets_instances");
}

extern "C" int pcnn_pack_pose_meta_fwd(const float* poses, const int32_t* cls, const float* intrinsics, int B, int I, float im_scale,
                                       int flip_x, float* pose_blob, int32_t* num_rows, float* meta, void* stream)
{
    PCNN_REQUIRE(poses && cls && intrinsics && pose_blob && num_rows && meta, "pack_pose_meta: NULL tensor pointer");
    PCNN_REQUIRE(B >= 1 && I >= 1 && B * I <= 1024, "pack_pose_meta: at most 1024 instance slots per batch (got %d x %d)", B, I);
    k_pack_pose_meta<<<1, 256, 0, (cudaStream_t)stream>>>(poses, cls, intrinsics, B, I, im_scale, flip_x, pose_blob, num_rows, meta);
    return check_launch("pack_pose_meta");
}

extern "C" int pcnn_loss_cls_hard_raw_fwd(const float* score_raw, const float* prob, const int32_t* gt, int B, int H, int W, int C,
                                          float threshold, float* loss_out, void* workspace, size_t workspace_bytes, void* stream)
{
    PCNN_REQUIRE(score_raw && prob && gt && loss_out && workspace, "loss_cls_hard_raw: NULL tensor pointer");
    PCNN_REQUIRE((unsigned long long)B * H * W < 0xffffffffULL, "loss_cls_hard_raw: too many pixels");
    size_t need = 0;
    pcnn_train_loss_workspace_bytes(&need);
    PCNN_REQUIRE(workspace_bytes >= need, "loss_cls_hard_raw: workspace too small (%zu < %zu)", workspace_bytes, need);
    double* partial = (double*)workspace;
    unsigned* ticket = (unsigned*)(partial + 2 * kLossBlocks);
    k_loss_cls_hard_raw<<<kLossBlocks, kLossThreads, 0, (cudaStream_t)stream>>>(score_raw, prob, gt, (unsigned)B * H * W, C, threshold, partial, ticket,
                                                                                loss_out);
    return check_launch("loss_cls_hard_raw");
}
