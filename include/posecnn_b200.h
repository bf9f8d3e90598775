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
/* the same im2col view of the RGB-D network's depth blob, formed from a RAW depth image [B,H,W] f32 (sensor units) with
 * the operation sequence of pcnn_conv1_depth_fused_tc (clip(d / 2000, 0, 1) * 255 tiled x3 - mean, float32 like numpy):
 * the input of the conv1_1_p weight gradient */
int pcnn_im2col_depth(const float* depth, const float* mean3_host, void* out_bf16, int B, int H, int W, void* stream);
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
 *  pcnn_up8_heads_bwd_ex  gradient of loss_cls (Hardlabel-selected cross entropy through log-softmax and the ReLU of `score`) and of
 *                         loss_vertex (smooth L1 on the labelled pixels' own class) w.r.t. the low-resolution head tensor, formed from
 *                         the loss structure on the fly: d_sc [B,h,w,Cs], d_vt [B,h,w,Cv] bf16 (padding channels zero), dbias [4C]
 *                         (C = 2, C even in 6..50, or C = 9); the labelled pixels' vertex values come from vertex_pred [B,H,W,3C], or
 *                         with vertex_pred == NULL from the low-resolution head tensor `lowres` [B,h,w,4C] + bias_vertex [3C];
 *                         workspace >= 16 C B ceil(h / 16) ceil(w / S) bytes, S = 16 cells at C = 2 and 4 otherwise (4 C floats per CTA)
 *  pcnn_pose_chain_bwd    Averagedistance's bottom_diff through l2_normalize, * poses_weight and tanh -> d fc8 pre-activation (fp16)
 *  pcnn_sgd_momentum      accum = mu * accum + (gscale * grad + wd * w); w -= lr * accum; refreshed 16-bit tensor-core copy (kind 0 bf16, 1 fp16)
 *  pcnn_transpose16 / pcnn_half_to_float   layout / precision glue of the fully connected backward GEMMs
 */
int pcnn_add_up2_bf16(const void* a4_bf16, const void* a5_bf16, int B, int h, int w, int C, void* out_bf16, void* stream);
int pcnn_up2_bwd_bf16(const void* dadd_bf16, const void* y5_bf16, int B, int h, int w, int C, void* d5_bf16, void* stream);
int pcnn_pack_lowres(const void* sc_bf16, int Cs, const void* vt_bf16, int Cv, int B, int h, int w, int C, float* lowres, void* stream);
int pcnn_up8_heads_bwd_ex(const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out, float upstream_cls,
                          float threshold, const float* vertex_pred, const float* lowres, const float* bias_vertex, const float* centers,
                          const float* vertex_loss_out, float upstream_vertex, float w_inside, float sigma, int B, int h, int w, int C,
                          int Cs, int Cv, void* d_sc_bf16, void* d_vt_bf16, float* dbias, void* workspace, size_t workspace_bytes,
                          void* stream);
/* pcnn_up8_heads_bwd_coord  the same adjoint for the VERTEX_REG_3D networks: the vertex target of a weighted pixel (label c in 1..C-1,
 *      centers[b, c, 2] > 0) is its object coordinate vertmap [B,8h,8w,3] f32 scaled by extents [C,3] f32 (as
 *      pcnn_vertex_targets_3d_fwd); every other argument, check, output and the workspace are those of pcnn_up8_heads_bwd_ex. */
int pcnn_up8_heads_bwd_coord(const float* prob, const float* score, const int32_t* gt, const float* cls_loss_out, float upstream_cls,
                             float threshold, const float* vertex_pred, const float* lowres, const float* bias_vertex, const float* vertmap,
                             const float* centers, const float* extents, const float* vertex_loss_out, float upstream_vertex, float w_inside,
                             float sigma, int B, int h, int w, int C, int Cs, int Cv, void* d_sc_bf16, void* d_vt_bf16, float* dbias,
                             void* workspace, size_t workspace_bytes, void* stream);
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
 * Domain-adaptation branch (networks/vgg16_convs.py:202-212, loss fcn/train.py:508-513), csrc/domain.cu:
 *   pool_score -> gradient_reversal(lambda) -> fc9 (25088 -> 256, ReLU) -> domain_score = fc(2) WITH ReLU (Network.fc's
 *   default, network.py:393,420) -> softmax -> argmax.  fc9 itself runs on pcnn_fc_f16_tc / pcnn_fc_dgrad_f16_tc /
 *   pcnn_fc_wgrad_f16_tc.
 *  pcnn_domain_tail   one launch over rows <= PCNN_HOUGH_MAX_ROWS: fc9_f16 [rows, ld] (fc9's fp16 output, 256 units, ld % 8 == 0,
 *      16-byte aligned), w10 [2][256] f32 (the domain_score weights, output-major), b10 [2] -> domain_score, domain_prob [rows, 2]
 *      f32 (score after its ReLU), domain_label [rows] int32 (first maximum on ties).  label_domain [rows] int32 (Hough's
 *      top_domain) may be NULL (inference: the gradient outputs are not touched).  With labels:
 *        loss[0] = loss_scale * sum_rows (logsumexp(z) - z[label]);  loss_scale = ADAPT_WEIGHT / (global row count);
 *        g = loss_scale * (softmax(z) - onehot(label)) * [z > 0];  dw10 [2][256] = g^T fc9;  db10 [2] = sum_rows g;
 *        d = (g @ w10) * [fc9 > 0];  db9 [256] = sum_rows d;  amax[0] = max |d|;
 *        dpre9_f16 [rows, ld] = grad_scale * d in fp16 (saturating at +-65504; columns >= 256 zero): the operand of fc9's
 *        backward GEMMs, loss-scaled by the caller's power of two grad_scale (the gradients sit below fp16's normal range).
 *      Every sum over rows runs in a fixed order: two launches give bit-identical outputs.
 *  pcnn_domain_grad_merge   dst[i] = scale_a * a[i] + scale_b * b[i] (fp32 products rounded, then added; n % 8 == 0, 16-byte
 *      aligned): the gradient of pool_score from the pose head (a = fc6's fp16 input gradient, scale_a = 1 / S) and the domain
 *      branch (b = fc9's, scale_b = -lambda / S_d: the gradient reversal).  With b = 0 it equals pcnn_half_to_float(a, scale_a).
 */
int pcnn_domain_tail(const void* fc9_f16, int rows, int ld, const float* w10, const float* b10, const int32_t* label_domain,
                     float loss_scale, float grad_scale, float* domain_score, float* domain_prob, int32_t* domain_label,
                     float* loss, float* amax, float* dw10, float* db10, float* db9, void* dpre9_f16, void* stream);
int pcnn_domain_grad_merge(const void* a_f16, float scale_a, const void* b_f16, float scale_b, size_t n, float* dst, void* stream);

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
/* 2 <= C <= 128, either parity.  vertex == NULL: label-only mode (label_2d / prob / score only; see pcnn_hough_vote_fwd_ex for the
 * consumer) */
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
 * Training-side target generation and the training step's two dense-head losses (SURVEY.md 8(f) rank 3).
 *  pcnn_vertex_targets_fwd     lib/gt_synthesize_layer/minibatch.py:543-602 (_generate_vertex_targets, single-instance
 *      branch): label [B,H,W] int32, centers [B,C,3] = (cx, cy, z) of each class's projected centre (z <= 0: class
 *      absent from the image) -> vertex_targets / vertex_weights [B,H,W,3C] f32 (zero elsewhere); float64 arithmetic
 *      rounded to float32 like numpy's (float32 centre - int64 pixel grid).
 * The losses (their gradients are the up-sampling adjoint's, pcnn_up8_heads_bwd_ex / _coord):
 *  pcnn_loss_cls_hard_raw_fwd  loss_cls, lib/fcn/train.py:455-465 over the Hardlabel selection (hard_label_op_gpu.cu.cc:16-29) on
 *      the raw `score` [B,H,W,C]: loss_out[0] = -sum_{selected p} log_softmax(score[p])[gt_p] / (count + 1e-10),
 *      loss_out[1] = count; neither the log-softmax nor the mask is materialised (declared above, with the backward kernels).
 *  pcnn_vertex_loss_fused_lowres_fwd / pcnn_vertex_loss_coord_lowres_fwd (below)   loss_vertex, lib/fcn/train.py:564-573
 *      (smooth_l1_loss_vertex) on the 2-D or the 3-D targets: loss_out[0] = sum(in_loss) / (sum(weights) + 1e-10),
 *      loss_out[1] = sum(weights).
 * Each reduces per-CTA partial sums (double) in index order: run-to-run deterministic.  workspace: zero-filled
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
/* the vertex loss on the targets / weights of pcnn_vertex_targets_fwd(label, centers, w_inside) WITHOUT materialising them
 * (5.2 GB at batch 32), with the vertex head given as the 1/8-resolution head tensor `lowres` [B,H/8,W/8,4C] + the vertex_pred
 * bias [3C] (values formed on demand with k_up8_heads' operation sequence: bit-identical to the dense tensor); H, W % 8 == 0 */
int pcnn_vertex_loss_fused_lowres_fwd(const float* lowres, const float* bias_vertex, const int32_t* label, const float* centers, int B,
                                      int H, int W, int C, float w_inside, float sigma, float* loss_out, void* workspace,
                                      size_t workspace_bytes, void* stream);
/* VERTEX_REG_3D targets (the 3-D branch of _generate_vertex_targets, minibatch.py:595-600, and _scale_vertmap, :605-616):
 *  pcnn_vertex_targets_3d_fwd   label [B,H,W] int32, vertmap [B,H,W,3] f32 (the object coordinate of each pixel, metres in the model
 *      frame), centers [B,C,3] (only z > 0 is read: the class is listed in the frame), extents [C,3] f32 -> vertex_targets /
 *      vertex_weights [B,H,W,3C] f32: for a pixel labelled c in 1..C-1 with a listed class, channel 3c+k = a_k * v_k + b_k with
 *      vmin = -e_k / 2, vmax = e_k / 2, a_k = 1 / (vmax - vmin), b_k = -vmin / (vmax - vmin) (a_k = b_k = 0 where vmax - vmin <= 0),
 *      all in float32 with the product rounded before the sum; weight w_inside on those channels; zero elsewhere.
 *  pcnn_vertex_loss_coord_lowres_fwd   pcnn_vertex_loss_fused_lowres_fwd on that target, without materialising it (same
 *      outputs and workspace). */
int pcnn_vertex_targets_3d_fwd(const int32_t* label, const float* vertmap, const float* centers, const float* extents, int B, int H, int W,
                               int C, float w_inside, float* targets, float* weights, void* stream);
int pcnn_vertex_loss_coord_lowres_fwd(const float* lowres, const float* bias_vertex, const int32_t* label, const float* vertmap,
                                      const float* centers, const float* extents, int B, int H, int W, int C, float w_inside, float sigma,
                                      float* loss_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Training image blobs (csrc/augment.cu): the image side of the synthetic-data loader, lib/gt_synthesize_layer/minibatch.py:147-200
 * with lib/utils/blob.py:74-129 (chromatic_transform, add_noise), PIXEL_MEANS subtraction (minibatch.py:179-180).
 * params [B, PCNN_AUG_PARAMS] f64 (device), one row per image, columns PCNN_AUG_*:
 *   BACKGROUND  background pool index; -1 (or any value outside [0, N)) = none: alpha == 0 pixels become 0 (minibatch.py:160-168)
 *   CHROMATIC   1 = run chromatic_transform with D_H / D_L / D_S, 0 = skip it
 *   NOISE       0 none, 1 Gaussian (SIGMA), 2 motion blur (BLUR_SIZE odd in 3..15, BLUR_AXIS 0 = along the row, 1 = along the column)
 * keys [B] u64: the image's Philox4x32-10 key; the Gaussian field g(pixel) = Box-Muller(Philox(key, pixel index)) belongs to the image,
 * so any shard of a batch produces the same rows.  noise_field [B,H,W] f64 (optional) replaces g bit for bit.
 *  pcnn_augment_color_fwd   rgba [B,H,W,channels] u8 (channels 4, or 3 = no alpha, no compositing), backgrounds [N,H,W,3] u8 ->
 *      blob [B,H,W,3] f32, per pixel: composite; BGR->HLS (OpenCV's uint8 arithmetic), H' = trunc((h + d_h) mod 180), L' / S' =
 *      trunc(clip(. + d, 0, 255)) in f64, HLS->BGR (OpenCV); Gaussian: clip(x + sigma g, 0, 255) in f64, one g for the three
 *      channels; blur: round(sum_{|t| <= r} x[reflect101(p + t)] / size) on the uint8 image; f32(f64(f32(x)) - mean3).
 *  pcnn_depth_blob_train_fwd   depth [B,H,W] u16 (depth_is_u16) or f32 -> depth_max [B] f32 = max(d) per image, blob [B,H,W,3]
 *      f32 = f32(f32(d) / max) * 255 tiled x3 (minibatch.py:187-200), the same noise on float data (blur: the float64 sum of the
 *      taps / size, rounded once), - mean3; its own params / keys (the reference draws add_noise again).  An all-zero image gives NaN
 *      (0 / 0), as numpy does.
 * mean3_host: 3 host doubles (PIXEL_MEANS, BGR).  A malformed params row never faults (unknown noise = none, size outside [1, 15]
 * = 1 tap).  No allocation, no host synchronisation; CUDA-graph capturable.
 */
#define PCNN_AUG_BACKGROUND 0
#define PCNN_AUG_CHROMATIC 1
#define PCNN_AUG_DH 2
#define PCNN_AUG_DL 3
#define PCNN_AUG_DS 4
#define PCNN_AUG_NOISE 5
#define PCNN_AUG_SIGMA 6
#define PCNN_AUG_BLUR_SIZE 7
#define PCNN_AUG_BLUR_AXIS 8
#define PCNN_AUG_PARAMS 9
int pcnn_augment_color_fwd(const uint8_t* rgba, int channels, const uint8_t* backgrounds, int num_backgrounds, const double* params,
                           const uint64_t* keys, const double* noise_field, int B, int H, int W, const double* mean3_host, float* blob,
                           void* stream);
int pcnn_depth_blob_train_fwd(const void* depth, int depth_is_u16, const double* params, const uint64_t* keys, const double* noise_field,
                              int B, int H, int W, const double* mean3_host, float* depth_max, float* blob, void* stream);

/* ---------------------------------------------------------------------------------------
 * Pose refinement with depth (csrc/pose_refine.cu, DESIGN.md 12): the ICP stage of lib/fcn/test.py:1314-1351
 * (Synthesizer::icp_python / solveICP) on the model point table, batched over every ROI row of a batch.
 *  label [B,H,W] int32, depth [B,H,W] f32 raw sensor units (z = depth / depth_factor), meta [B, num_meta] (fx = m[0],
 *  px = m[2], fy = m[4], py = m[5]), rois / poses [cap,7] (image = rois[r,0] - batch_offset, class = rois[r,1]),
 *  num_rows: device int32 (NULL = cap), points [C,P,3] (P <= 4096).
 *  -> poses_refined [cap,7] (depth re-centring along the ray), poses_icp [cap,7] (best of 8 depth hypotheses after `iterations`
 *  point-to-plane Gauss-Newton steps), info [cap,4] = (class pixels, chosen hypothesis, score, inliers at its final pose),
 *  trace [cap, 8, iterations + 1, 8] (nullable) = per hypothesis and step the pose (7) and its inlier count.
 *  Rows with class <= 0 or >= C, image outside [0,B), r >= *num_rows or fewer than min_pixels class pixels are zero (info[0] =
 *  the class pixel count).  workspace: pcnn_pose_refine_workspace_bytes.  Deterministic, no host synchronisation. */
int pcnn_pose_refine_workspace_bytes(int B, int C, size_t* bytes);
int pcnn_pose_refine_fwd(const int32_t* label, const float* depth, const float* meta, int num_meta, const float* rois,
                         const float* poses, const int32_t* num_rows, int cap, const float* points, int C, int P, int B, int H, int W,
                         int batch_offset, float depth_factor, float znear, float zfar, float max_error, int min_pixels,
                         int iterations, float* poses_refined, float* poses_icp, float* info, float* trace, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Pose estimation from object coordinates and depth (csrc/coord_pose.cu, DESIGN.md 13): the VERTEX_REG_3D test path,
 * Synthesizer::estimatePose3D (lib/synthesize/synthesize.cpp:1769-1966), batched.
 *  label [B,H,W] int32; object coordinates scaled into [0,1] by the class extents from the dense vertex [B,H,W,3C], or (vertex
 *  NULL) evaluated at the sampled pixels from lowres [B,H/8,W/8,4C] + bias_vertex [3C] like the Hough entry; depth [B,H,W] f32 raw
 *  sensor units (0 = hole, z = depth / depth_factor); meta [B, num_meta] (fx = m[0], px = m[2], fy = m[4], py = m[5]); extents
 *  [C,3]; keys [B]: the per-image Philox4x32-10 keys.  2 <= C <= 128.
 *  -> poses [B,C,3,4] ([R | t] per class, zero where no pose was found; class 0 unused), info [B,C,6] = (class pixels,
 *  hypotheses drawn for the class, inliers of the survivor at its last count, final energy or -1, hypotheses of the image that
 *  hit the attempt cap, survivor's hypothesis index or -1).  trace_hyp [B,256,13] (nullable) = per hypothesis (class or 0,
 *  attempts, three pixel indices or -1, inlier count in each of the 8 rounds or -1); trace_round [B,C,8,4] (nullable) = per
 *  class and round (pixels taken, their index sum mod 2^32, best hypothesis, its inliers).  workspace:
 *  pcnn_coord_pose3d_workspace_bytes.  Deterministic, no host synchronisation.  There is no batch_offset: an image's result
 *  depends only on its own inputs and keys[b], so a shard of a batch passes the slices of the inputs and of the keys (the offset
 *  only numbers the records, pcnn_coord_pose3d_records).
 * pcnn_coord_pose3d_records: the detection records of lib/fcn/test.py:1383-1399 from poses [B,C,3,4]: for every image and class
 *  j >= 1 with t_z > 0, in (image, class) order, rois [B*(C-1),6] = (image + batch_offset, j, _get_bb2D(extent, pose, K) *
 *  im_scale) with K = the meta intrinsics / im_scale (meta holds K * im_scale), poses [B*(C-1),7] = (mat2quat(R), t); rows after
 *  the last are zero, *num_rows (device int32) = the row count. */
int pcnn_coord_pose3d_workspace_bytes(int B, int H, int W, int C, size_t* bytes);
int pcnn_coord_pose3d_fwd(const int32_t* label, const float* vertex, const float* lowres, const float* bias_vertex, const float* depth,
                          const float* meta, int num_meta, const float* extents, const uint64_t* keys, int B, int H, int W, int C,
                          float depth_factor, float* poses, float* info, int32_t* trace_hyp, int32_t* trace_round, void* workspace,
                          size_t workspace_bytes, void* stream);
int pcnn_coord_pose3d_records(const float* poses, const float* extents, const float* meta, int num_meta, int B, int C, int batch_offset,
                              float im_scale, float* rois, float* out_poses, int32_t* num_rows, void* stream);

/* Colour-only pose estimation from object coordinates (csrc/coord_pose.cu, DESIGN.md 13): Synthesizer::estimatePose2D
 * (lib/synthesize/synthesize.cpp:1571-1767), batched; the arguments of pcnn_coord_pose3d_fwd without depth and depth_factor.
 *  Hypotheses from four pixels by P3P, inliers within 10 px of the projection; the survivor keeps its P3P pose (no refit, no
 *  Nelder-Mead, as the reference behaves).  -> poses [B,C,3,4], info [B,C,6] as pcnn_coord_pose3d_fwd with energy = -1;
 *  trace_hyp [B,256,14] (nullable) = per hypothesis (class or 0, attempts, four pixel indices or -1, inlier count in each of the
 *  8 rounds or -1); trace_round [B,C,8,4] (nullable) as pcnn_coord_pose3d_fwd.  workspace: pcnn_coord_pose2d_workspace_bytes.
 *  The records come from pcnn_coord_pose3d_records.  Deterministic, no host synchronisation. */
int pcnn_coord_pose2d_workspace_bytes(int B, int H, int W, int C, size_t* bytes);
int pcnn_coord_pose2d_fwd(const int32_t* label, const float* vertex, const float* lowres, const float* bias_vertex, const float* meta,
                          int num_meta, const float* extents, const uint64_t* keys, int B, int H, int W, int C, float* poses, float* info,
                          int32_t* trace_hyp, int32_t* trace_round, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Evaluation of the test-time records (csrc/evaluate.cu, DESIGN.md 14): the scorer of lib/datasets/lov.py:397-680 and
 * linemod.py:626-760 on the device.  Every output accumulates (the caller zeroes it once); counts are int64; 2 <= C <= 128.
 *  pcnn_eval_confusion   gt_label, label [num_pixels] int32 -> hist [C,C] += the confusion matrix of fast_hist
 *      (datasets/imdb.py:123-125): row = gt, column = prediction; a pixel counts only when 0 <= gt < C.  A prediction outside
 *      [0, C) is an argument error: it is not counted, and status[0] += the number of such pixels.
 *  pcnn_eval_pose_errors   scores 1 to 4 pose sets (poses0..3 [cap,7] = (qw,qx,qy,qz, tx,ty,tz), sharing rois [cap, roi_stride]
 *      with image = rois[:,0], class = rois[:,1]) against gt_rows [num_gt,14] = (image, class, [R | t] 3x4 row-major).
 *      Rows k < *num_rows (NULL = cap; a value outside [0, cap] is clamped and counts in status[1]).  Pairing as lov.py:576-628:
 *      every gt j with 0 < class < C counts once in counts[s][0][class] (count_all) and pairs with every row of the same image and
 *      class; pairs are gt-major, rows ascending, so duplicate detections each form a pair.  A gt of a foreground class whose
 *      image - batch_offset is outside [0, B) is not scored and counts in status[1].
 *      Per pair p < *num_pairs: pairs [num_gt*cap, 2] = (j, k); per set s: errors [s][p] = (re deg, te, ADD or ADD-S, reproj px)
 *      f64, flags [s][p] = bit0 error < threshold[class] (counts[s][1][class] += 1), bit1 reproj < 5 px (counts[s][2][class] += 1),
 *      bit2 the eggbox flip was applied.  symmetric [C] > 0: ADD-S (adi); flip_z [C] > 0: an estimate more than 90 degrees off is
 *      scored for reprojection as R diag(-1,-1,1) (linemod.py:727-733).  K = meta[image - batch_offset, 0:9]; points [C,P,3],
 *      P <= 4096; num_gt <= 4096.  counts [num_sets,3,C].  Deterministic, no host synchronisation, CUDA-graph capturable.
 *  pcnn_eval_gt_rows_from_blob   pose_blob [n,13] (image, class, box, qw,qx,qy,qz, tx,ty,tz) -> gt_rows [n,14], R by quat2mat.
 */
int pcnn_eval_confusion(const int32_t* gt_label, const int32_t* label, size_t num_pixels, int C, int64_t* hist, int64_t* status,
                        void* stream);
int pcnn_eval_pose_errors(const float* gt_rows, int num_gt, const float* rois, int roi_stride, int cap, const int32_t* num_rows,
                          const float* poses0, const float* poses1, const float* poses2, const float* poses3, int num_sets,
                          const float* meta, int num_meta, int B, int batch_offset, const float* points, int C, int P,
                          const float* symmetric, const float* threshold, const float* flip_z, int32_t* pairs, double* errors,
                          int32_t* flags, int32_t* num_pairs, int64_t* counts, int64_t* status, void* stream);
int pcnn_eval_gt_rows_from_blob(const float* pose_blob, int n, float* gt_rows, void* stream);

/* ---------------------------------------------------------------------------------------
 * Image scale (csrc/rescale.cu, DESIGN.md 15): cv2.resize(x, None, None, fx=fx, fy=fx, interpolation) of the SCALES_BASE != 1
 * configurations (the LINEMOD *_3d.yml models use 1.5), batched NHWC, with OpenCV's generic (non-SIMD) arithmetic bit for bit:
 *   LINEAR   coordinate f = float((d + 0.5) / fx - 0.5) in double, s = floor(f), a = f - s; columns clamp s to [0, W - 1] with
 *            a = 0 there, rows clamp only the two row indices; two float32 lerps with every product and sum rounded (no FMA).
 *   NEAREST  s = min(floor(d * (1 / fx)), n - 1) in double.
 * The destination [B,Ho,Wo,...] must be Ho = round(H * fx), Wo = round(W * fx) (half to even, as cv2 sizes it), else
 * PCNN_E_INVALID; so must a row whose W * C or Wo * C elements overflow int (the kernels' in-row index).  B <= 65535.
 *  pcnn_resize_color_u8     the test-time colour blob (fcn/test.py:49-65): frames [B,H,W,3] u8 BGR -> blob [B,Ho,Wo,3] f32, the
 *      source value f32(f64(u8) - mean3_host[c]) (numpy's float64 PIXEL_MEANS), resized LINEAR.
 *  pcnn_resize_linear_f32   LINEAR on [B,H,W,C] f32, C = 1 or 3: the training colour blob after augmentation and PIXEL_MEANS
 *      (gt_synthesize_layer/minibatch.py:179-183) and the object-coordinate vertmap (minibatch.py:416).
 *  pcnn_resize_depth        LINEAR on the raw depth [B,H,W] (fcn/test.py:1335, 1384): u16 (depth_is_u16) or f32 holding integer
 *      sensor units; the result, of the input's type, is rounded half to even and saturated to [0, 65535] as cv2's uint16 output.
 *  pcnn_resize_nearest_i32  NEAREST on label maps [B,H,W] int32: the training label image (minibatch.py:352) and the predicted
 *      labels back to the frame with fx = 1 / s (fcn/test.py:1421).
 * One CTA per output row; no allocation, no host synchronisation; CUDA-graph capturable. */
int pcnn_resize_color_u8(const uint8_t* frames, int B, int H, int W, double fx, int Ho, int Wo, const double* mean3_host, float* blob,
                         void* stream);
int pcnn_resize_linear_f32(const float* src, int B, int H, int W, int C, double fx, int Ho, int Wo, float* dst, void* stream);
int pcnn_resize_depth(const void* depth, int depth_is_u16, int B, int H, int W, double fx, int Ho, int Wo, void* dst, void* stream);
int pcnn_resize_nearest_i32(const int32_t* label, int B, int H, int W, double fx, int Ho, int Wo, int32_t* dst, void* stream);

/* ---------------------------------------------------------------------------------------
 * Detection network at test time (csrc/det.cu, DESIGN.md 16): networks/vgg16_det.py:94-137, from conv_rpn to the fc6 operand.
 *  pcnn_rpn_heads_fwd   conv_rpn [npix,512] bf16 x weights [6A][512] bf16 (rows 0..2A-1 rpn_cls_score, 2A..6A-1 rpn_bbox_pred;
 *      output-major) + bias [6A] f32, fp32 accumulation on the tensor cores; both 1x1 convolutions keep Network.conv's ReLU
 *      (network.py:160).  -> cls_prob [npix,2A] f32 = the pair softmax of reshape_score (channel a against channel A + a,
 *      network.py:700-710; foreground = channels A..2A-1), bbox_pred [npix,4A] f32 (ReLU'd deltas, anchor-major).  1 <= A <= 64.
 *  pcnn_rpn_proposals_fwd   rpn_layer/proposal_layer.py for each of B images: cls_prob [B,h,w,2A], bbox_pred [B,h,w,4A], anchors
 *      [h*w*A,4] f32 (snippets.py:generate_anchors_pre, order (h, w, a)); bbox_transform_inv + clip_boxes to [0, im_w - 1] x
 *      [0, im_h - 1] in fp32 with numpy's operation order (no FMA); the K = min(pre_top_n, h*w*A) best anchors in the canonical
 *      order (descending foreground probability, ties by ascending anchor index; the reference's unstable argsort leaves ties
 *      unordered); greedy NMS with nms_kernel.cu's devIoU (+1 areas, fp32, no FMA), suppressing IoU > nms_thresh; the first
 *      post_top_n kept boxes.  -> rois [B*post_top_n,5] (b, x1, y1, x2, y2), scores [B*post_top_n] and num_rois [B] int32;
 *      rows past num_rois[b] are (b, 0, 0, 0, 0) with score 0.  pre_boxes [B*K,5] (nullable): the sorted, decoded, clipped
 *      candidates (x1, y1, x2, y2, score) NMS ran on.  1 <= A <= 64, 1 <= pre_top_n <= 16384, post_top_n >= 1.  workspace:
 *      pcnn_rpn_proposals_workspace_bytes (B * K * (20 + 8 * ceil(K / 64)) bytes, the NMS bitmask).
 *  pcnn_crop_pool_f16   network.py:791-809: each ROI (b, x1, y1, x2, y2) of rois [N, roi_stride] divided by ((H-1) * feat_stride,
 *      (W-1) * feat_stride), tf.image.crop_and_resize (TF 1.x bilinear: in_y = y1 * (H-1) + y * (y2-y1) * (H-1) / 13, samples
 *      outside [0, H-1] x [0, W-1] are 0) to 14 x 14 on feat [B,H,W,C] bf16, then max_pool2d 2 x 2 / 2 -> out [N, 7*7*C] fp16
 *      (h, w, c), saturated to +-65504.  fp32, every product and sum rounded.  A batch index outside [0, B) crops zeros.  C % 8 == 0.
 *  pcnn_softmax_rows_f32   out[r] = softmax(in[r]) over cols (cls_prob = softmax(cls_score)).
 *  pcnn_det_records_fwd   the test loop's records (fcn/test.py:1589-1616, 1639-1691, 1731-1746) for B images of `rows` proposal
 *      rows each: cls_prob [B*rows,C], bbox_pred [B*rows,4C] (normalised deltas), poses_tanh [B*rows,4C], rois [B*rows,5]
 *      (b, x1, y1, x2, y2), num_rois [B] int32 (rows r < num_rois[b] count).  For each class j = 1..C-1 of image b, slot
 *      b*(C-1) + j-1: the row with the top cls_prob[:, j] > 0.02f (ties: the lowest row; NaN never), its box de-normalised
 *      (f32(f64(d) * (0.1, 0.1, 0.2, 0.2))), bbox_transform_inv'd and clipped to [0, im_w-1] x [0, im_h-1] in fp32 without FMA,
 *      and the depth z of compute_translations' Nelder-Mead fit (scipy 1.18.1 at N = 1, x0 = 0.5, at most 200 evaluations) of
 *      the projected points [C,P,3] of class j (R = quat2mat(q) in fp64 rounded to fp32, fp32 camera coordinates, K =
 *      f64(meta[b, 0:9]) in fp64) to the box's width and height.  -> dets [B*(C-1),7] (b, j, x1, y1, x2, y2, score), poses
 *      [B*(C-1),7] (q raw, f32(rx z), f32(ry z), f32(z)), trace [B*(C-1),2] int32 (iterations, evaluations), num_dets [B] int32
 *      (zeroed here, then counted).  An empty slot is (b, 0, 0, 0, 0, 0, 0) with a zero pose and trace.  2 <= C <= 128,
 *      1 <= P <= 4096, 1 <= B <= 65535, num_meta >= 9.
 * No allocation, no host synchronisation; CUDA-graph capturable. */
int pcnn_rpn_heads_fwd(const void* conv_rpn_bf16, const void* weights_bf16, const float* bias, int npix, int A, float* cls_prob,
                       float* bbox_pred, void* stream);
int pcnn_rpn_proposals_workspace_bytes(int B, int h, int w, int A, int pre_top_n, size_t* bytes);
int pcnn_rpn_proposals_fwd(const float* cls_prob, const float* bbox_pred, const float* anchors, int B, int h, int w, int A, float im_h,
                           float im_w, int pre_top_n, int post_top_n, float nms_thresh, float* rois, float* scores, int32_t* num_rois,
                           float* pre_boxes, void* workspace, size_t workspace_bytes, void* stream);
int pcnn_crop_pool_f16(const void* feat_bf16, int B, int H, int W, int C, const float* rois, int num_rois, int roi_stride,
                       float feat_stride, void* out_f16, void* stream);
int pcnn_softmax_rows_f32(const float* in, int rows, int cols, float* out, void* stream);
int pcnn_det_records_fwd(const float* cls_prob, const float* bbox_pred, const float* poses_tanh, const float* rois,
                         const int32_t* num_rois, int B, int rows, int C, int im_h, int im_w, const float* meta, int num_meta,
                         const float* points, int P, float* dets, float* poses, int32_t* num_dets, int32_t* trace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* POSECNN_B200_H_ */
