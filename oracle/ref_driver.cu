// ref_driver.cu — C entry points around the reference's OWN CUDA kernels.
//
// TEST INFRASTRUCTURE ONLY.  Each section #includes one of the reference's *_gpu.cu.cc files
// from where it lies under /root/reference (never copied into this repo) and compiles it
// unmodified for sm_90a behind oracle/ref_shim.  The result (oracle/_ref/libposecnn_ref.so)
// is the "second oracle" of SURVEY.md §8(c): it pins the CPU restatement
// (oracle/posecnn_oracle.c) and produces the golden vectors under tests/golden/.
// One section per translation unit: compile with -DREF_SECTION=<n> (see oracle/Makefile).
#define REF_STR2(x) #x
#define REF_STR(x) REF_STR2(x)
#define REF_FILE(rel) REF_STR(REF_ROOT/lib/rel)

#include "ref_shim.h"

static Eigen::GpuDevice g_dev;
static tensorflow::OpKernelContext g_ctx;

#if REF_SECTION == 1  // ------------------------------------------------------------- Hough
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/sort.h>
#include REF_FILE(hough_voting_gpu_layer/hough_voting_gpu_op.cu.cc)

// The op exactly as the reference runs it (HoughvotinggpuOp<GpuDevice>::Compute,
// hough_voting_gpu_op.cc:321-428): reset, per-image launcher, row count.  Non-deterministic
// list order inside (atomicAdd compaction); with skip_pixels = 1 the vote SET is order free.
extern "C" int ref_hough_full(const int* label, const float* vertex, const float* extents, const float* meta,
                              const float* gt, int B, int H, int W, int C, int num_gt, int num_meta, int is_train,
                              float vote_thr, float per_thr, int skip, float* top_box, float* top_pose,
                              float* top_target, float* top_weight, int* top_domain, int* num_rois_dev,
                              int* num_rois_host)
{
    ::reset_outputs(top_box, top_pose, top_target, top_weight, top_domain, num_rois_dev, C);
    for (int n = 0; n < B; n++) {
        HoughVotingLaucher(&g_ctx, label + (size_t)n * H * W, vertex + (size_t)n * H * W * 3 * C, extents,
                           meta + (size_t)n * num_meta, gt, n, B, H, W, C, num_gt, is_train, 0.9f, 500, vote_thr, per_thr,
                           skip, top_box, top_pose, top_target, top_weight, top_domain, num_rois_dev, g_dev);
        g_ctx.release_all();
    }
    ::copy_num_rois(num_rois_host, num_rois_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

// Canonical run: the reference kernels (compute_arrays_kernel, compute_hough_kernel,
// compute_max_indexes_kernel, compute_rois_kernel) driven with per-class pixel lists sorted
// into ascending pixel order (SURVEY.md §8(c) canonicalisation).  The host flow between the
// kernels restates HoughVotingLaucher (.cu.cc:615-797).  votes_out: optional [B][C][H][W].
extern "C" int ref_hough_canonical(const int* label, const float* vertex, const float* extents, const float* meta_all,
                                   const float* gt, int B, int H, int W, int C, int num_gt, int num_meta, int is_train,
                                   float vote_thr, float per_thr, int skip, float* top_box, float* top_pose,
                                   float* top_target, float* top_weight, int* top_domain, int* num_rois_dev,
                                   int* num_rois_host, float* votes_out)
{
    const int T = 1024, HW = H * W;
    ::reset_outputs(top_box, top_pose, top_target, top_weight, top_domain, num_rois_dev, C);
    if (votes_out) cudaMemset(votes_out, 0, sizeof(float) * (size_t)B * C * HW);
    int *arrays, *sizes, *cls_idx, *max_idx, *num_max;
    float *hspace, *hdata;
    cudaMalloc(&arrays, sizeof(int) * (size_t)C * HW);
    cudaMalloc(&sizes, sizeof(int) * C);
    cudaMalloc(&cls_idx, sizeof(int) * C);
    cudaMalloc(&max_idx, sizeof(int) * (size_t)C * HW);
    cudaMalloc(&num_max, sizeof(int));
    cudaMalloc(&hspace, sizeof(float) * (size_t)C * HW);
    cudaMalloc(&hdata, sizeof(float) * (size_t)C * HW * 3);
    std::vector<int> sizes_h(C), cls_h(C);
    const int index_size = 128 / B;
    for (int n = 0; n < B; n++) {
        const int* lab = label + (size_t)n * HW;
        const float* vert = vertex + (size_t)n * HW * 3 * C;
        const float* meta = meta_all + (size_t)n * num_meta;
        cudaMemset(sizes, 0, sizeof(int) * C);
        compute_arrays_kernel<<<(HW + T - 1) / T, T>>>(HW, lab, arrays, sizes, H, W);
        cudaMemcpy(sizes_h.data(), sizes, sizeof(int) * C, cudaMemcpyDeviceToHost);
        int count = 0;
        for (int c = 1; c < C; c++)
            if (sizes_h[c] > 500) cls_h[count++] = c;
        if (count == 0) continue;
        for (int i = 0; i < count; i++) {  // canonical order
            thrust::device_ptr<int> p(arrays + (size_t)cls_h[i] * HW);
            thrust::sort(thrust::device, p, p + sizes_h[cls_h[i]]);
        }
        cudaMemcpy(cls_idx, cls_h.data(), sizeof(int) * count, cudaMemcpyHostToDevice);
        cudaMemset(hspace, 0, sizeof(float) * (size_t)count * HW);
        cudaMemset(hdata, 0, sizeof(float) * (size_t)count * HW * 3);
        int out = count * HW;
        compute_hough_kernel<<<(out + T - 1) / T, T>>>(out, hspace, hdata, lab, vert, extents, meta, arrays, sizes, cls_idx,
                                                       H, W, C, count, 0.9f, skip);
        if (votes_out)
            for (int i = 0; i < count; i++)
                cudaMemcpy(votes_out + ((size_t)n * C + cls_h[i]) * HW, hspace + (size_t)i * HW, sizeof(float) * HW,
                           cudaMemcpyDeviceToDevice);
        int nmax = 0;
        if (vote_thr > 0) {
            cudaMemset(num_max, 0, sizeof(int));
            compute_max_indexes_kernel<<<(out + T - 1) / T, T>>>(out, max_idx, C * HW, num_max, hspace, hdata, H, W,
                                                                 vote_thr, per_thr);
            cudaMemcpy(&nmax, num_max, sizeof(int), cudaMemcpyDeviceToHost);
            thrust::device_ptr<int> p(max_idx);
            thrust::sort(thrust::device, p, p + nmax);  // canonical: ascending flat index
        } else {
            std::vector<int> mh(count);
            for (int i = 0; i < count; i++) {
                float* hm = thrust::max_element(thrust::device, hspace + (size_t)i * HW, hspace + (size_t)(i + 1) * HW);
                mh[i] = (int)(hm - hspace);
            }
            cudaMemcpy(max_idx, mh.data(), sizeof(int) * count, cudaMemcpyHostToDevice);
            nmax = count;
        }
        if (nmax >= index_size) nmax = index_size;
        // one thread at a time so that rows come out in canonical order
        for (int i = 0; i < nmax; i++)
            compute_rois_kernel<<<1, 1>>>(1, top_box, top_pose, top_target, top_weight, top_domain, extents, meta, gt,
                                          hspace, hdata, max_idx + i, cls_idx, is_train, n, H, W, C, num_gt, num_rois_dev);
    }
    ::copy_num_rois(num_rois_host, num_rois_dev);
    cudaFree(arrays); cudaFree(sizes); cudaFree(cls_idx); cudaFree(max_idx); cudaFree(num_max); cudaFree(hspace);
    cudaFree(hdata);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { fprintf(stderr, "ref_hough_canonical: %s\n", cudaGetErrorString(e)); return -1; }
    return 0;
}

#elif REF_SECTION == 2  // ----------------------------------------------------------- RoiPool
#include REF_FILE(roi_pooling_layer/roi_pooling_op_gpu.cu.cc)
extern "C" int ref_roi_pool_fwd(const float* bottom, const float* rois, int num_rois, int channel_rois, int height,
                                int width, int channels, int ph, int pw, float scale, int pool_channel, float* top,
                                int* argmax)
{
    ::ROIPoolForwardLaucher(bottom, scale, pool_channel, num_rois, channel_rois, height, width, channels, ph, pw, rois, top,
                          argmax, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
extern "C" int ref_roi_pool_bwd(const float* top_diff, const int* argmax, const float* rois, int batch, int num_rois,
                                int channel_rois, int height, int width, int channels, int ph, int pw, float scale,
                                int pool_channel, float* bottom_diff)
{
    ::ROIPoolBackwardLaucher(top_diff, scale, pool_channel, batch, num_rois, channel_rois, height, width, channels, ph, pw,
                           rois, bottom_diff, argmax, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

#elif REF_SECTION == 3  // ----------------------------------------------------------- Hardlabel
#include REF_FILE(hard_label_layer/hard_label_op_gpu.cu.cc)
extern "C" int ref_hard_label_fwd(const float* prob, const int* gt, int B, int H, int W, int C, float thr, float* top)
{
    ::HardlabelForwardLaucher(prob, gt, B, H, W, C, thr, top, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

#elif REF_SECTION == 4  // ----------------------------------------------------------- Backproject
#include REF_FILE(backprojecting_layer/backprojecting_op_gpu.cu.cc)
extern "C" int ref_backproject_fwd(const float* data, const float* label, const float* depth, const float* meta,
                                   const float* label_3d, int B, int H, int W, int Cf, int C, int num_meta, int G, int ks,
                                   float thr, float* top_data, float* top_label, float* top_flag)
{
    ::BackprojectForwardLaucher(data, label, depth, meta, label_3d, B, H, W, Cf, C, num_meta, G, ks, thr, top_data, top_label,
                              top_flag, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
extern "C" int ref_backproject_bwd(const float* top_diff, const float* depth, const float* meta, int B, int H, int W,
                                   int Cf, int num_meta, int G, float* bottom_diff)
{
    ::BackprojectBackwardLaucher(top_diff, depth, meta, B, H, W, Cf, num_meta, G, bottom_diff, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

#elif REF_SECTION == 5  // ----------------------------------------------------------- Project
#include REF_FILE(projecting_layer/projecting_op_gpu.cu.cc)
extern "C" int ref_project_fwd(const float* data, const float* depth, const float* meta, int B, int H, int W, int Cf,
                               int num_meta, int G, float* top)
{
    ::ProjectForwardLaucher(data, depth, meta, B, H, W, Cf, num_meta, G, top, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
extern "C" int ref_project_bwd(const float* top_diff, const float* depth, const float* meta, int B, int H, int W, int Cf,
                               int num_meta, int G, int ks, float thr, float* bottom_diff)
{
    ::ProjectBackwardLaucher(top_diff, depth, meta, B, H, W, Cf, num_meta, G, ks, thr, bottom_diff, g_dev);
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

#elif REF_SECTION == 6  // ----------------------------------------------------------- Averagedistance
#include REF_FILE(average_distance_loss/average_distance_loss_op_gpu.cu.cc)
extern "C" int ref_average_distance_fwd(const float* pred, const float* target, const float* weight, const float* point,
                                        const float* symmetry, int N, int C, int P, float margin, float* loss,
                                        float* bottom_diff)
{
    ::AveragedistanceForwardLaucher(&g_ctx, pred, target, weight, point, symmetry, N, C, P, margin, loss, bottom_diff, g_dev);
    g_ctx.release_all();
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
#endif
