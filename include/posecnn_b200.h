/*
 * posecnn_b200.h — C ABI of libposecnn_b200.so (hand-written sm_90a CUDA).
 *
 * One entry point per native launcher of the reference (yuxng/PoseCNN @ 9f3dd7b).  The
 * reference's launchers take raw device pointers + ints + an Eigen::GpuDevice; these take
 * raw device pointers + ints + a cudaStream_t (passed as void*), so a TF1 OpKernel::Compute,
 * a PyTorch extension or a ctypes caller can bind them without any framework type.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - tensors are dense, row-major, NHWC, float32 / int32 — exactly the reference layouts;
 *   - the caller owns all memory, including the workspace (size from *_workspace_bytes);
 *   - all work is enqueued on `stream`; no entry point synchronises or allocates;
 *   - return value: 0 = success, negative = error (PCNN_E_*); pcnn_last_error() returns a
 *     thread-local message.  Nothing ever calls exit() (the reference does, e.g.
 *     lib/hough_voting_gpu_layer/hough_voting_gpu_op.cu.cc:679-684).
 *
 * Citations are relative to /root/reference/lib.
 */
#ifndef POSECNN_B200_H_
#define POSECNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCNN_OK 0
#define PCNN_E_INVALID (-1)   /* bad argument (rank/shape/attr), like OP_REQUIRES -> InvalidArgument */
#define PCNN_E_WORKSPACE (-2) /* workspace too small */
#define PCNN_E_CUDA (-3)      /* CUDA runtime error at launch */

#define PCNN_MAX_ROI 128                       /* hough_voting_gpu_op.cu.cc:14 */
#define PCNN_HOUGH_MAX_ROWS (PCNN_MAX_ROI * 9) /* hough_voting_gpu_op.cc:94 */

const char* pcnn_last_error(void);
int pcnn_version(void);

/* ---------------------------------------------------------------------------------------
 * Houghvotinggpu — replaces HoughvotinggpuOp<GpuDevice>::Compute + HoughVotingLaucher
 * (hough_voting_gpu_layer/hough_voting_gpu_op.cc:299-435, hough_voting_gpu_op.cu.cc:615-797;
 * registration hough_voting_gpu_op.cc:37-52).  Whole batch per call, no host round trips.
 *
 *   label   [B,H,W] int32          vertex [B,H,W,3C] f32        extents [C,3] f32
 *   meta    [B,num_meta] f32       gt [num_gt,13] f32 (may be NULL when num_gt == 0)
 * Outputs are CAPACITY buffers of PCNN_HOUGH_MAX_ROWS rows, zero-filled by the call:
 *   top_box [1152,7]  top_pose [1152,7]  top_target [1152,4C]  top_weight [1152,4C]
 *   top_domain [1152] int32   num_rois [1] int32 = number of valid rows (the op reports
 *   max(1, num_rois) rows, hough_voting_gpu_op.cc:379-383; the Python layer applies that rule).
 * Hard-coded reference constants are explicit parameters with the same defaults:
 *   inlier_threshold 0.9, label_threshold 500 (hough_voting_gpu_op.cc:356-357).
 * Canonical order (the reference is non-deterministic, SURVEY.md §8(c)): per-class pixel
 * lists in ascending pixel index; maxima in ascending (class, cell) order; rows ordered by
 * image then maximum.
 * status (optional, [4] int32, device): [0] bit0 = candidate list overflow (threshold mode),
 * [1] = number of selected cells whose interval-scan vote differed from the per-cell recount.
 */
int pcnn_hough_vote_workspace_bytes(int B, int H, int W, int C, int skip_pixels, float threshold_vote,
                                    size_t* bytes);
int pcnn_hough_vote_fwd(const int32_t* label, const float* vertex, const float* extents, const float* meta,
                        const float* gt, int B, int H, int W, int C, int num_gt, int num_meta, int is_train,
                        float inlier_threshold, int label_threshold, float threshold_vote,
                        float threshold_percentage, int skip_pixels, float* top_box, float* top_pose,
                        float* top_target, float* top_weight, int32_t* top_domain, int32_t* num_rois,
                        int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
/* Extended form of pcnn_hough_vote_fwd for the two things a caller that owns the whole pipeline needs:
 *  (1) image shards of a larger batch (SURVEY.md 8(e)): this call holds images [batch_offset, batch_offset + B) of a
 *      batch of batch_global images; the ROI budget is MAX_ROI / batch_global per image (hough_voting_gpu_op.cu.cc:733,
 *      applied to the batch the reference op would see), top_box[:,0] and the gt match use GLOBAL batch indices, so
 *      the concatenation of the shards' rows in rank order equals the single-call result on the whole batch;
 *  (2) vertex == NULL: the sampled pixels' (dx, dy, log z) are computed on demand from the network's 1/8-resolution head
 *      tensor `lowres` [B,H/8,W/8,4C] (pcnn_lowres_heads) + bias_vertex [3C] with pcnn_up8_heads' own operation
 *      sequence — bit-identical to reading the dense vertex_pred, which then never has to be written (2.6 GB per
 *      batch of 32).  With vertex != NULL, lowres / bias_vertex are ignored. */
int pcnn_hough_vote_fwd_ex(const int32_t* label, const float* vertex, const float* lowres, const float* bias_vertex,
                           const float* extents, const float* meta, const float* gt, int B, int batch_global,
                           int batch_offset, int H, int W, int C, int num_gt, int num_meta, int is_train,
                           float inlier_threshold, int label_threshold, float threshold_vote,
                           float threshold_percentage, int skip_pixels, float* top_box, float* top_pose,
                           float* top_target, float* top_weight, int32_t* top_domain, int32_t* num_rois,
                           int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
/* Debug / parity helper: dense vote planes [B,C,H,W] f32 (0 for classes that did not vote),
 * computed by the same interval-scan kernels.  Used by tests to compare with the oracle. */
int pcnn_hough_vote_planes(const int32_t* label, const float* vertex, const float* extents, const float* meta,
                           int B, int H, int W, int C, int num_meta, float inlier_threshold,
                           int label_threshold, int skip_pixels, float* votes, void* workspace,
                           size_t workspace_bytes, void* stream);
/* HoughvotinggpuGrad (hough_voting_gpu_op.cu.cc:608-612): zeros for label [B,H,W] (as f32)
 * and vertex [B,H,W,3C]. */
int pcnn_hough_vote_bwd(float* grad_label, float* grad_vertex, int B, int H, int W, int C, void* stream);

/* ---------------------------------------------------------------------------------------
 * RoiPool / RoiPoolGrad — replaces ROIPoolForwardLaucher / ROIPoolBackwardLaucher
 * (roi_pooling_layer/roi_pooling_op_gpu.cu.cc:103-131, 232-253; registration
 * roi_pooling_op.cc:29-50).  bottom [B,H,W,Cc]; rois [N,channel_rois] rows
 * [b, cls, x1,y1,x2,y2,...]; top/argmax [N,ph,pw,Cc] (or 1 channel when pool_channel).
 */
int pcnn_roi_pool_fwd(const float* bottom, const float* rois, int num_rois, int channel_rois, int batch,
                      int height, int width, int channels, int pooled_height, int pooled_width,
                      float spatial_scale, int pool_channel, float* top, int32_t* argmax, void* stream);
/* same forward reading bf16 NHWC features (the tensor-core trunk's activation format); channels % 8 == 0 */
int pcnn_roi_pool_fwd_bf16(const void* bottom_bf16, const float* rois, int num_rois, int channel_rois, int batch,
                           int height, int width, int channels, int pooled_height, int pooled_width,
                           float spatial_scale, float* top, int32_t* argmax, void* stream);
int pcnn_roi_pool_bwd(const float* top_diff, const int32_t* argmax, const float* rois, int batch, int num_rois,
                      int channel_rois, int height, int width, int channels, int pooled_height,
                      int pooled_width, float spatial_scale, int pool_channel, float* bottom_diff,
                      void* stream);

/* ---------------------------------------------------------------------------------------
 * Hardlabel / HardlabelGrad — replaces HardlabelForwardLaucher / HardlabelBackwardLaucher
 * (hard_label_layer/hard_label_op_gpu.cu.cc:32-51, 66-84; registration hard_label_op.cc:30-44).
 * prob [B,H,W,C] f32, gt [B,H,W] int32 -> top [B,H,W,C] f32.
 */
int pcnn_hard_label_fwd(const float* prob, const int32_t* gt, int B, int H, int W, int C, float threshold,
                        float* top, void* stream);
int pcnn_hard_label_bwd(int B, int H, int W, int C, float* grad_prob, float* grad_gt, void* stream);

/* ---------------------------------------------------------------------------------------
 * Backproject / BackprojectGrad — replaces BackprojectForwardLaucher / BackwardLaucher
 * (backprojecting_layer/backprojecting_op_gpu.cu.cc:128-155, 221-241; registration
 * backprojecting_op.cc:30-53).  data [B,H,W,Cf], label [B,H,W,C], depth [B,H,W],
 * meta [B,num_meta], label_3d [B,G,G,G,C] -> top_data [B,G,G,G,Cf], top_label [B,G,G,G,C],
 * top_flag [B,G,G,G,Cf] (Cf channels, backprojecting_op.cc:363-369).
 */
int pcnn_backproject_fwd(const float* data, const float* label, const float* depth, const float* meta,
                         const float* label_3d, int B, int H, int W, int Cf, int C, int num_meta,
                         int grid_size, int kernel_size, float threshold, float* top_data, float* top_label,
                         float* top_flag, void* stream);
int pcnn_backproject_bwd(const float* top_diff, const float* depth, const float* meta, int B, int H, int W,
                         int Cf, int num_meta, int grid_size, float* bottom_diff, void* stream);

/* ---------------------------------------------------------------------------------------
 * Project / ProjectGrad — replaces ProjectForwardLaucher / ProjectBackwardLaucher
 * (projecting_layer/projecting_op_gpu.cu.cc:76-98, 172-192; registration projecting_op.cc:30-47).
 * data [B,G,G,G,Cf], depth [B,H,W], meta [B,num_meta] -> top [B,H,W,Cf].
 */
int pcnn_project_fwd(const float* data, const float* depth, const float* meta, int B, int H, int W, int Cf,
                     int num_meta, int grid_size, float* top, void* stream);
int pcnn_project_bwd(const float* top_diff, const float* depth, const float* meta, int B, int H, int W, int Cf,
                     int num_meta, int grid_size, int kernel_size, float threshold, float* bottom_diff,
                     void* stream);

/* ---------------------------------------------------------------------------------------
 * Averagedistance / AveragedistanceGrad — replaces AveragedistanceForwardLaucher /
 * AveragedistanceBackwardLaucher (average_distance_loss/average_distance_loss_op_gpu.cu.cc:256-343,
 * 357-377; registration average_distance_loss_op.cc:38-54).
 * prediction/target/weight [N,4C], point [C,P,3], symmetry [C] -> loss [1], bottom_diff [N,4C].
 * One launch, no host synchronisation; workspace = N+64 floats (the reference allocates
 * N*P*(54+4C+1) scratch floats and reduces through thrust + a host copy, .cu.cc:268-335).
 */
int pcnn_average_distance_workspace_bytes(int N, size_t* bytes);
int pcnn_average_distance_fwd(const float* prediction, const float* target, const float* weight,
                              const float* point, const float* symmetry, int N, int C, int P, float margin,
                              float* loss, float* bottom_diff, void* workspace, size_t workspace_bytes,
                              void* stream);
int pcnn_average_distance_bwd(const float* top_diff, const float* bottom_diff, int N, int channels,
                              float* output, void* stream);

/* ---------------------------------------------------------------------------------------
 * VGG16 convolution stack on the tensor cores — replaces Network.conv / Network.max_pool
 * (networks/network.py:159-188, 303-310: tf.nn.conv2d NHWC x HWIO, SAME, stride 1, bias, ReLU;
 * 2x2/2 max pool) as wired by networks/vgg16_convs.py:80-97, 128-163.
 * Implicit GEMM on wgmma (BF16 operands, FP32 accumulation in registers, TMA-fed, im2col folded
 * into the TMA box coordinates).  Activations are NHWC bf16; weights are [Cout][k*k*Cin] bf16
 * (tap-major, channel-minor; converted once from the TF HWIO layout).  block_n = 0 picks the
 * N tile (64 / 128 / 256) from Cout.
 */
int pcnn_conv_bf16_tc(const void* in_bf16, const void* weights_bf16, const float* bias, void* out_bf16, int B,
                      int H, int W, int Cin, int Cout, int ksize, int relu, int block_n, void* stream);
/* same with the following 2x2 / stride-2 max pool (network.py:303-310) fused into the epilogue: out = [B,H/2,W/2,Cout] */
int pcnn_conv_pool_bf16_tc(const void* in_bf16, const void* weights_bf16, const float* bias, void* out_pooled_bf16,
                           int B, int H, int W, int Cin, int Cout, int ksize, int relu, int block_n, void* stream);
/* conv1_1 (Cin = 3): in [B,H,W,Cin] f32, weights HWIO [3,3,Cin,Cout] f32 -> out [B,H,W,Cout] bf16 */
int pcnn_conv3x3_small_cin(const float* in, const float* weights_hwio, const float* bias, void* out_bf16, int B,
                           int H, int W, int Cin, int Cout, int relu, void* stream);
/* first layer on the tensor cores: im2col [B,H,W,3] (f32, or u8 minus per-channel mean: the BGR - PIXEL_MEANS
 * pre-processing of lib/fcn/test.py:37-110 fused) -> [B,H,W,64] bf16 with K = tap*3 + c, then a 1x1 pcnn_conv_bf16_tc */
int pcnn_im2col_c3(const void* in, int in_is_u8, const float* mean3_host, void* out_bf16, int B, int H, int W,
                   void* stream);
/* conv1_1 with the im2col built in shared memory (no HBM round trip): in [B,H,W,3] u8 (minus mean) or f32,
 * weights [64][64] bf16 in the K order tap*3 + c (zero padded), bias [64] -> out [B,H,W,64] bf16 */
int pcnn_conv1_fused_tc(const void* in, int in_is_u8, const float* mean3_host, const void* weights_bf16,
                        const float* bias, void* out_bf16, int B, int H, int W, int relu, void* stream);
/* conv1_1_p of the RGB-D network on a RAW depth image: depth [B,H,W] f32 (sensor units); the depth blob
 * clip(d / 2000, 0, 1) * 255 tiled x3 - PIXEL_MEANS (lib/fcn/test.py:70-76) is formed in the loader, float32 like numpy */
int pcnn_conv1_depth_fused_tc(const float* depth, const float* mean3_host, const void* weights_bf16, const float* bias,
                              void* out_bf16, int B, int H, int W, int relu, void* stream);
int pcnn_maxpool2x2_bf16(const void* in_bf16, void* out_bf16, int B, int H, int W, int C, void* stream);

/* ---------------------------------------------------------------------------------------
 * Backward pass of the convolution / fully connected layers for the training step (lib/fcn/train.py:206-260 drives
 * TensorFlow's gradients of Network.conv / Network.fc / Network.max_pool, networks/network.py:159-188, 303-310, 392-422):
 *   dz = dy * [y > 0];  dW[r,s,ci,co] = sum_{n,h,w} x[n,h+r-1,w+s-1,ci] * dz[n,h,w,co];  db = sum dz;
 *   dx = conv(dz, W flipped and transposed) = pcnn_conv_bf16_tc on conv.hwio_to_tc_dgrad weights.
 *  pcnn_conv_wgrad_bf16_tc   weight gradient on wgmma with BOTH operands MN-major (the reduction index = pixel is the row of
 *      the NHWC activation tiles as TMA delivers them: no transposed copies), split-K over pixel ranges with a fixed-order
 *      reduction; x [B,H,W,Cin], dz [B,H,W,Cout] bf16 -> dW [Cout][ksize*ksize*Cin] f32 (the tensor-core weight layout) =
 *      scale * gradient (+ decay * w when w != NULL: the l2_regularizer term, network.py:171-172).  A fully connected layer is
 *      the 1x1 case with B = H = 1, W = rows.  Cin, Cout multiples of 64.
 *  pcnn_relu_bwd_bf16 / pcnn_maxpool_relu_bwd_bf16   dz from the upstream gradient and the layer's stored output (ReLU mask;
 *      2x2/2 max-pool routing to the window's first maximum fused with the mask of the conv below), optionally the bias
 *      gradient db [C] = scale * sum_pixels dz (+ decay * b) through per-CTA partials in bias_ws (pcnn_bias_ws_bytes).
 *  pcnn_add_to_bf16          gradient fan-in: out = a + b (+ b_f32), bf16 out.
 */
int pcnn_conv_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, size_t* bytes);
int pcnn_conv_wgrad_bf16_tc(const void* x_bf16, const void* dz_bf16, int B, int H, int W, int Cin, int Cout, int ksize,
                            float scale, const float* w_f32, float decay, float* dW, void* workspace, size_t workspace_bytes,
                            void* stream);
/* fully connected layer: x [rows, Cin], dy [rows, Cout] fp16 -> dW [Cout][Cin] f32; workspace: pcnn_conv_wgrad_workspace_bytes(1, 1, rows, Cin, Cout, 1) */
int pcnn_fc_wgrad_f16_tc(const void* x_f16, const void* dy_f16, int rows, int Cin, int Cout, float scale, const float* w_f32,
                         float decay, float* dW, void* workspace, size_t workspace_bytes, void* stream);
int pcnn_bias_ws_bytes(int C, size_t* bytes);
int pcnn_relu_bwd_bf16(const void* g_bf16, const void* y_bf16, size_t npix, int C, int has_relu, void* dz_bf16, float scale,
                       const float* b, float decay, float* db, void* bias_ws, size_t bias_ws_bytes, void* stream);
int pcnn_maxpool_relu_bwd_bf16(const void* g_bf16, const void* y_bf16, int B, int H, int W, int C, void* dz_bf16, float scale,
                               const float* b, float decay, float* db, void* bias_ws, size_t bias_ws_bytes, void* stream);
int pcnn_add_to_bf16(const void* a_bf16, const void* b_bf16, const float* b_f32, size_t n, void* out_bf16, void* stream);

/* Small kernels of the training step around those GEMMs (csrc/train_bwd.cu); training graph lib/networks/vgg16_convs.py:128-212,
 * losses lib/fcn/train.py:455-465, 564-573, optimizer tf.train.MomentumOptimizer (train.py:633):
 *  pcnn_add_up2_bf16 / pcnn_up2_bwd_bf16   add = a4 + up2(a5) (fixed bilinear conv2d_transpose 4x4 / 2) and its adjoint (+ ReLU mask of a5)
 *  pcnn_pack_lowres       [score C | vertex 3C] f32 head tensor from the two bf16 1x1-convolution outputs (row strides Cs, Cv)
 *  pcnn_up8_heads_bwd     gradient of loss_cls (Hardlabel-selected cross entropy through log-softmax and the ReLU of `score`) and of
 *                         loss_vertex (smooth L1 on the labelled pixels' own class) w.r.t. the low-resolution head tensor, formed from
 *                         the loss structure on the fly: d_sc [B,h,w,Cs], d_vt [B,h,w,Cv] bf16 (padding channels zero), dbias [4C]
 *  pcnn_pose_chain_bwd    Averagedistance's bottom_diff through l2_normalize, * poses_weight and tanh -> d fc8 pre-activation (fp16)
 *  pcnn_sgd_momentum      accum = mu * accum + (gscale * grad + wd * w); w -= lr * accum; refreshed 16-bit tensor-core copy (kind 0 bf16, 1 fp16)
 *  pcnn_transpose16 / pcnn_half_to_float   layout / precision glue of the fully connected backward GEMMs
 *  pcnn_conv1_wgrad       conv1_1 weight gradient (Cin = 3) on the CUDA cores, input = uint8 image - mean
 */
int pcnn_add_up2_bf16(const void* a4_bf16, const void* a5_bf16, int B, int h, int w, int C, void* out_bf16, void* stream);
int pcnn_up2_bwd_bf16(const void* dadd_bf16, const void* y5_bf16, int B, int h, int w, int C, void* d5_bf16, void* stream);
int pcnn_pack_lowres(const void* sc_bf16, int Cs, const void* vt_bf16, int Cv, int B, int h, int w, int C, float* lowres, void* stream);
int pcnn_up8_heads_bwd(const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out, float upstream_cls,
                       float threshold, const float* vertex_pred, const float* centers, const float* vertex_loss_out,
                       float upstream_vertex, float w_inside, float sigma, int B, int h, int w, int C, int Cs, int Cv,
                       void* d_sc_bf16, void* d_vt_bf16, float* dbias, void* workspace, size_t workspace_bytes, void* stream);
/* the same with vertex_pred == NULL: the labelled pixels' vertex values are formed from the low-resolution head tensor
 * `lowres` [B,h,w,4C] + bias_vertex [3C] (no dense vertex_pred in the training step; C = 22) */
int pcnn_up8_heads_bwd_ex(const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out, float upstream_cls,
                          float threshold, const float* vertex_pred, const float* lowres, const float* bias_vertex, const float* centers,
                          const float* vertex_loss_out, float upstream_vertex, float w_inside, float sigma, int B, int h, int w, int C,
                          int Cs, int Cv, void* d_sc_bf16, void* d_vt_bf16, float* dbias, void* workspace, size_t workspace_bytes,
                          void* stream);
int pcnn_pose_chain_bwd(const float* bottom_diff, const float* poses_tanh, const float* poses_weight, int N, int D, float upstream,
                        void* dpre_f16, int ld, void* stream);
int pcnn_sgd_momentum(float* w, float* accum, const float* grad, size_t n, float lr, float mu, float wd, float gscale, void* copy16,
                      int kind, void* stream);
/* loss_cross_entropy_single_frame on the Hardlabel selection from the RAW `score` layer (log-softmax per selected pixel) */
int pcnn_loss_cls_hard_raw_fwd(const float* score_raw, const float* prob, const int32_t* gt, int B, int H, int W, int C,
                               float threshold, float* loss_out, void* workspace, size_t workspace_bytes, void* stream);
/* input gradient of a fully connected layer: out [M, ld_out] fp16 = (dy [M,K] @ W[N,K]^T) * [relu_mask > 0]; W = the layer's weights in
 * TF layout [in = N][out = K] fp16 (K contiguous); relu_mask [M, ld_out] fp16 = stored output of the ReLU layer below, or NULL */
int pcnn_fc_dgrad_f16_tc(const void* dy_f16, const void* w_in_out_f16, int M, int N, int K, const void* relu_mask_f16, void* out_f16,
                         int ld_out, void* workspace, size_t workspace_bytes, void* stream);
int pcnn_transpose16(const void* in, int rows, int cols, void* out, void* stream);
int pcnn_half_to_float(const void* src_f16, size_t n, float scale, float* dst, void* stream);
int pcnn_conv1_wgrad(const void* img_u8, const float* mean3_host, const void* dz_bf16, int B, int H, int W, float scale,
                     const float* w, float decay, float* dW, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Pose-regression head (networks/vgg16_convs.py:177-197, Network.fc networks/network.py:392-422, tanh :436-438) on own
 * kernels (csrc/fc_tc.cu); inference path (no argmax, no gradients).
 *  pcnn_roi_pool_pair_f16  pool_score = RoiPool(conv5_3, scale5) + RoiPool(conv4_3, scale4) with the RoiPool rule of
 *      roi_pooling_layer/roi_pooling_op_gpu.cu.cc:19-101, added in fp32 and written as the fp16 fc6 operand
 *      [num_rois, pooled_h*pooled_w*C] in (h, w, c) order.  f5 [B,H5,W5,C], f4 [B,H4,W4,C] bf16 NHWC; rois
 *      [num_rois, roi_stride] f32 rows [batch, cls, x1,y1,x2,y2,...]; the image index is rois[:,0] - batch_offset
 *      (image shards carry global batch indices); an index outside [0, B) pools nothing (zeros).
 *  pcnn_fc_f16_tc          out = act(A[M,K] @ W[N,K]^T + bias): wgmma GEMM, FP16 operands (11-bit mantissa: the 1e-3 quaternion tolerance), FP32 accumulation, split-K
 *      over the grid with a fixed-order reduction (deterministic); A, W fp16 row-major with K contiguous, N % 128 == 0,
 *      K % 64 == 0; rows n_valid..N of W are zero padding; act 0 none / 1 ReLU / 2 tanh; outputs: out_f16 [M, ld_out]
 *      (optional) and / or out_f32 [M, n_valid] (optional).  workspace: pcnn_fc_workspace_bytes(M, N, K).
 */
int pcnn_roi_pool_pair_f16(const void* f5_bf16, int H5, int W5, const void* f4_bf16, int H4, int W4, int C, int B,
                            int batch_offset, const float* rois, int num_rois, int roi_stride, int pooled_h,
                            int pooled_w, float scale5, float scale4, void* out_f16, void* stream);
int pcnn_fc_workspace_bytes(int M, int N, int K, size_t* bytes);
int pcnn_fc_f16_tc(const void* a_f16, const void* w_f16, const float* bias, int M, int N, int K, int n_valid, int act,
                   void* out_f16, int ld_out, float* out_f32, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * FCN heads after the 1x1 convolutions on conv4_3 / conv5_3 (networks/vgg16_convs.py:128-163):
 * add + fixed-bilinear conv2d_transpose (networks/network.py:141-157, 207-222) + `score` /
 * `vertex_pred` 1x1 + softmax / arg-max.  The bilinear up-sampling commutes with the 1x1
 * convolutions, so the matrices are applied at 1/8 resolution (pcnn_lowres_heads) and one
 * streaming kernel (pcnn_up8_heads) produces label_2d [B,H,W] int32, vertex_pred [B,H,W,3C] f32
 * and (optional) prob_normalized / score [B,H,W,C] f32.
 *   score4/vert4 [B,h,w,Cs|Cv] bf16 (1x1 convs of conv4_3), score5/vert5 [B,h/2,w/2,Cs|Cv] bf16,
 *   w_score [Cs][C] f32, w_vertex [Cv][3C] f32, lowres [B,h,w,4C] f32, H = 8h, W = 8w.
 *   w_vertex == NULL: "folded" vertex head -- the caller multiplied the vertex_pred matrix into the two vertex 1x1
 *   convolutions (linear, no ReLU between them: vgg16_convs.py:151-163), vert4 / vert5 then hold the 3C vertex
 *   channels directly (row stride Cv >= 3C, zero padded) and the kernel only adds and up-samples them.
 */
int pcnn_lowres_heads(const void* score4, const void* score5, const void* vert4, const void* vert5,
                      const float* w_score, const float* w_vertex, int B, int h, int w, int Cs, int Cv, int C,
                      float* lowres, void* stream);
/* vertex == NULL: label-only mode (label_2d / prob / score only; see pcnn_hough_vote_fwd_ex for the consumer) */
int pcnn_up8_heads(const float* lowres, const float* bias_score, const float* bias_vertex, int B, int h, int w,
                   int C, int32_t* label, float* vertex, float* prob, float* score, void* stream);
/* depthwise bilinear conv2d_transpose (k x k, stride s, SAME) on f32 NHWC — un-fused reference path */
int pcnn_deconv_bilinear(const float* in, float* out, int B, int h, int w, int C, int k, int s, void* stream);

/* ---------------------------------------------------------------------------------------
 * Test-time post-processing on the device (SURVEY.md 8(f) rank 1) — replaces lib/utils/nms.py:3-32
 * `nms(rois, 0.5)` and the pose assembly loop of lib/fcn/test.py:197-211:
 *   greedy NMS in descending score order (ties: larger row index first = stable argsort reversed); a box is dropped
 *   when IoU(+1 convention, fp32) > thresh with a kept box of the same class (per_image = 1: and the same image; the
 *   reference ignores the batch column and only runs batch 1, per_image = 0 reproduces that);
 *   out_rois[k] = rois[keep[k]], out_poses[k] = [poses_pred[keep[k], 4c:4c+4] | poses_init[keep[k], 4:7]];
 *   keep is in processing order (per_image = 1: image by image, ascending batch index, processing order inside an image).
 * rois [capacity,7], poses_init [capacity,7], poses_pred [capacity,4C] or NULL (then poses_init is passed through);
 * rows considered: max(*num_rois_dev, 1) when num_rois_dev != NULL (Hough's device row count; the reference always has
 * the dummy row), else num_rows.  Outputs are capacity buffers (rows beyond *num_keep are zero, keep = -1): no host
 * synchronisation, CUDA-graph capturable.  capacity <= PCNN_HOUGH_MAX_ROWS.
 */
int pcnn_nms_pose_fwd(const float* rois, const float* poses_init, const float* poses_pred, const int* num_rois_dev,
                      int num_rows, int capacity, int num_classes, float thresh, int per_image, int32_t* keep,
                      float* out_rois, float* out_poses, int32_t* num_keep, void* stream);

/* ---------------------------------------------------------------------------------------
 * Training-side target generation and fused losses (SURVEY.md 8(f) rank 3).
 *  pcnn_vertex_targets_fwd     lib/gt_synthesize_layer/minibatch.py:543-602 (_generate_vertex_targets, single-instance
 *      branch): label [B,H,W] int32, centers [B,C,3] = (cx, cy, z) of each class's projected centre (z <= 0: class
 *      absent from the image) -> vertex_targets / vertex_weights [B,H,W,3C] f32 (zero elsewhere); float64 arithmetic
 *      rounded to float32 like numpy's (float32 centre - int64 pixel grid).
 *  pcnn_loss_cls_hard_fwd      lib/fcn/train.py:455-465 on the Hardlabel mask (hard_label_op_gpu.cu.cc:16-29) without
 *      materialising it: loss = -sum_{selected p} score[p, gt_p] / (count + 1e-10), score = log-softmax [B,H,W,C];
 *      loss_out[0] = loss, loss_out[1] = count; grad_score (optional, [B,H,W,C]) = upstream * d loss / d score.
 *  pcnn_smooth_l1_vertex_fwd   lib/fcn/train.py:564-573: loss_out[0] = sum(in_loss) / (sum(weights) + 1e-10),
 *      loss_out[1] = sum(weights); grad_pred optional.
 * Both losses reduce per-CTA partial sums (double) in index order: run-to-run deterministic.  workspace: zero-filled
 * once by the caller (pcnn_train_loss_workspace_bytes), reusable across launches on one stream.
 */
/*  pcnn_vertex_targets_instances_fwd   the multi-instance branch of _generate_vertex_targets (minibatch.py:549-573): several
 *      instances of one class are separated by an instance-mask image; mask [B,H,W] int32, instances [B,I,5] f32 =
 *      (cls, mask id = cls_indexes_old + 1, cx, cy, z), z <= 0 = unused slot; a pixel with label == cls and mask == id gets
 *      the target toward that instance's centre (last matching instance wins, like the reference's in-order overwrites).
 *  pcnn_pack_pose_meta_fwd             the data layer's pose blob and meta_data packing (minibatch.py:440-451, 474-492):
 *      poses [B,I,12] (3x4 [R|T] row-major per instance), cls [B,I] int32 (< 0 = unused slot), intrinsics [B,9] ->
 *      pose_blob [B*I,13] rows [image, cls, 0,0,0,0, qw,qx,qy,qz (transforms3d mat2quat, w >= 0), tx,ty,tz] compacted in
 *      (image, slot) order, rows beyond *num_rows zero; meta [B,48] = K * im_scale (K[2][2] = 1) | its inverse | zeros,
 *      FLIP_X sign flips of minibatch.py:488-491.  One small launch each; no host synchronisation. */
int pcnn_vertex_targets_instances_fwd(const int32_t* label, const int32_t* mask, const float* instances, int B, int H, int W,
                                      int C, int I, float w_inside, float* targets, float* weights, void* stream);
int pcnn_pack_pose_meta_fwd(const float* poses, const int32_t* cls, const float* intrinsics, int B, int I, float im_scale,
                            int flip_x, float* pose_blob, int32_t* num_rows, float* meta, void* stream);
int pcnn_train_loss_workspace_bytes(size_t* bytes);
int pcnn_vertex_targets_fwd(const int32_t* label, const float* centers, int B, int H, int W, int C, float w_inside,
                            float* targets, float* weights, void* stream);
int pcnn_loss_cls_hard_fwd(const float* score, const float* prob, const int32_t* gt, int B, int H, int W, int C,
                           float threshold, float* loss_out, float upstream, float* grad_score, void* workspace,
                           size_t workspace_bytes, void* stream);
int pcnn_smooth_l1_vertex_fwd(const float* pred, const float* targets, const float* weights, size_t n, float sigma,
                              float* loss_out, float upstream, float* grad_pred, void* workspace, size_t workspace_bytes,
                              void* stream);
/* the same vertex loss WITHOUT materialising targets / weights (5.2 GB at batch 32): equals
 * pcnn_smooth_l1_vertex_fwd(pred, targets, weights) with (targets, weights) = pcnn_vertex_targets_fwd(label, centers,
 * w_inside); reads 12 bytes of pred per labelled pixel.  grad_pred (optional, dense [B,H,W,3C]) is zero-filled here. */
int pcnn_vertex_loss_fused_fwd(const float* pred, const int32_t* label, const float* centers, int B, int H, int W, int C,
                               float w_inside, float sigma, float* loss_out, float upstream, float* grad_pred,
                               void* workspace, size_t workspace_bytes, void* stream);
/* the same loss with the vertex head given as the 1/8-resolution head tensor `lowres` [B,H/8,W/8,4C] + the vertex_pred bias [3C]
 * (values formed on demand with k_up8_heads' operation sequence: bit-identical to the dense tensor) */
int pcnn_vertex_loss_fused_lowres_fwd(const float* lowres, const float* bias_vertex, const int32_t* label, const float* centers, int B,
                                      int H, int W, int C, float w_inside, float sigma, float* loss_out, void* workspace,
                                      size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* POSECNN_B200_H_ */
