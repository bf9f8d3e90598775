"""Host-side bindings of the pose-regression head kernels (include/posecnn_b200.h, csrc/fc_tc.cu):
RoiPool x2 + add (-> fp16 fc6 operand), and the fully connected layers as split-K wgmma GEMMs with fused
bias / ReLU / tanh (lib/networks/vgg16_convs.py:177-197, lib/networks/network.py:392-422); the training step's backward of
those layers (input and weight gradients, the pose-loss chain into fc8, and their layout / precision glue)."""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, lib, ptr, stream, workspace


def fc_weights_to_tc(w_in_out: torch.Tensor, dtype=torch.float16) -> torch.Tensor:
    """TF fc weights [in, out] f32 (network.py:404-406) -> [out padded to a multiple of 128][in] fp16 (or `dtype`; K contiguous)."""
    k, n = w_in_out.shape
    npad = (n + 127) // 128 * 128
    w = torch.zeros((npad, k), dtype=dtype, device=w_in_out.device)
    w[:n] = w_in_out.t().to(dtype)
    return w.contiguous()


def roi_pool_pair(f5: torch.Tensor, f4: torch.Tensor, rois: torch.Tensor, pooled_h: int = 7, pooled_w: int = 7,
                  scale5: float = 1.0 / 16.0, scale4: float = 1.0 / 8.0, batch_offset: int = 0) -> torch.Tensor:
    """[N, pooled_h * pooled_w * C] fp16 = RoiPool(f5, scale5) + RoiPool(f4, scale4), flattened (h, w, c)."""
    assert f5.is_cuda and f5.dtype == torch.bfloat16 and f5.is_contiguous() and f4.dtype == torch.bfloat16 and f4.is_contiguous()
    assert rois.is_cuda and rois.dtype == torch.float32 and rois.is_contiguous() and rois.dim() == 2
    B, H5, W5, C = f5.shape
    _, H4, W4, C4 = f4.shape
    assert C4 == C and f4.shape[0] == B
    n = rois.shape[0]
    out = torch.empty((n, pooled_h * pooled_w * C), dtype=torch.float16, device=f5.device)
    check(lib().pcnn_roi_pool_pair_f16(ptr(f5), H5, W5, ptr(f4), H4, W4, C, B, int(batch_offset), ptr(rois), n, rois.shape[1],
                                        int(pooled_h), int(pooled_w), scale5, scale4, ptr(out), stream()))
    return out


def crop_pool(feat: torch.Tensor, rois: torch.Tensor, feat_stride: float = 16.0) -> torch.Tensor:
    """crop_pool of the detection network (network.py:791-809): [N, 7 * 7 * C] fp16 = max_pool2d 2x2 of crop_and_resize to 14 x 14
    of feat [B,H,W,C] bf16 at the boxes rois [N,5] (b, x1, y1, x2, y2) in image pixels, flattened (h, w, c)."""
    assert feat.is_cuda and feat.dtype == torch.bfloat16 and feat.is_contiguous() and feat.dim() == 4
    assert rois.is_cuda and rois.dtype == torch.float32 and rois.is_contiguous() and rois.dim() == 2
    B, H, W, C = feat.shape
    n = rois.shape[0]
    out = torch.empty((n, 7 * 7 * C), dtype=torch.float16, device=feat.device)
    check(lib().pcnn_crop_pool_f16(ptr(feat), B, H, W, C, ptr(rois), n, rois.shape[1], float(feat_stride), ptr(out), stream()))
    return out


def softmax_rows(x: torch.Tensor) -> torch.Tensor:
    """softmax over the last dimension of x [rows, cols] f32 (cls_prob = softmax(cls_score))."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
    out = torch.empty_like(x)
    check(lib().pcnn_softmax_rows_f32(ptr(x), x.shape[0], x.shape[1], ptr(out), stream()))
    return out


def fc(a: torch.Tensor, w_tc: torch.Tensor, bias: torch.Tensor, act: str = "relu", out_dtype=torch.float16) -> torch.Tensor:
    """act(a @ w^T + bias).  a [M, K] fp16, w_tc = fc_weights_to_tc(W) [Npad, K] fp16, bias [n_valid] f32.
    out_dtype fp16 -> [M, Npad] (the next layer's operand; padding columns are zero), f32 -> [M, n_valid]."""
    assert a.is_cuda and a.dtype == torch.float16 and a.is_contiguous() and a.dim() == 2
    assert w_tc.dtype == torch.float16 and w_tc.is_contiguous() and bias.dtype == torch.float32
    M, K = a.shape
    N = w_tc.shape[0]
    assert w_tc.shape[1] == K
    nv = bias.numel()
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_fc_workspace_bytes(M, N, K, ctypes.byref(nbytes)))
    ws = workspace("fc", nbytes.value, a.device)
    code = {"none": 0, "relu": 1, "tanh": 2}[act]
    if out_dtype == torch.float16:
        out = torch.empty((M, N), dtype=torch.float16, device=a.device)
        check(lib().pcnn_fc_f16_tc(ptr(a), ptr(w_tc), ptr(bias), M, N, K, nv, code, ptr(out), N, ptr(None), ptr(ws), ws.numel(), stream()))
    else:
        out = torch.empty((M, nv), dtype=torch.float32, device=a.device)
        check(lib().pcnn_fc_f16_tc(ptr(a), ptr(w_tc), ptr(bias), M, N, K, nv, code, ptr(None), 0, ptr(out), ptr(ws), ws.numel(), stream()))
    return out


def fc_dgrad(dy: torch.Tensor, w_t: torch.Tensor, relu_mask: torch.Tensor | None) -> torch.Tensor:
    """Input gradient of a fully connected layer (pcnn_fc_dgrad_f16_tc): [M, N] fp16 = (dy [M, K] @ w_t^T) * [relu_mask > 0].
    w_t [N][K] fp16 = the layer's [in][out padded] weights (transpose16 of its fc_weights_to_tc copy); relu_mask [M, N] fp16 = the
    stored output of the ReLU layer below, or None."""
    M, K = dy.shape
    N = w_t.shape[0]
    out = torch.empty((M, N), dtype=torch.float16, device=dy.device)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_fc_workspace_bytes(M, N, K, ctypes.byref(nbytes)))
    ws = workspace("fc", nbytes.value, dy.device)
    check(lib().pcnn_fc_dgrad_f16_tc(ptr(dy), ptr(w_t), M, N, K, ptr(relu_mask), ptr(out), N, ptr(ws), ws.numel(), stream()))
    return out


def fc_wgrad(x: torch.Tensor, dy: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """Weight gradient of a fully connected layer (pcnn_fc_wgrad_f16_tc): [Cout][Cin] f32 = scale * dy^T @ x, x [rows, Cin] and
    dy [rows, Cout] fp16."""
    rows, Cin = x.shape
    Cout = dy.shape[1]
    out = torch.empty((Cout, Cin), dtype=torch.float32, device=x.device)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_conv_wgrad_workspace_bytes(1, 1, rows, Cin, Cout, 1, ctypes.byref(nbytes)))
    ws = workspace("wgrad", nbytes.value, x.device)
    check(lib().pcnn_fc_wgrad_f16_tc(ptr(x), ptr(dy), rows, Cin, Cout, scale, ptr(None), 0.0, ptr(out), ptr(ws), ws.numel(), stream()))
    return out


def pose_chain_bwd(bottom_diff: torch.Tensor, poses_tanh: torch.Tensor, poses_weight: torch.Tensor, upstream: float,
                   out: torch.Tensor) -> torch.Tensor:
    """pcnn_pose_chain_bwd: Averagedistance's bottom_diff [N, D] f32 through l2_normalize, * poses_weight and tanh, times upstream,
    written to out [N, ld] fp16 (fc8's d pre-activation; ld = fc8's padded output count, columns D.. written as 0).  Returns out."""
    N, D = bottom_diff.shape
    check(lib().pcnn_pose_chain_bwd(ptr(bottom_diff), ptr(poses_tanh), ptr(poses_weight), N, D, upstream, ptr(out), out.shape[1], stream()))
    return out


def transpose16(x: torch.Tensor) -> torch.Tensor:
    """pcnn_transpose16: x [rows, cols] (any 16-bit dtype) -> [cols, rows]."""
    rows, cols = x.shape
    out = torch.empty((cols, rows), dtype=x.dtype, device=x.device)
    check(lib().pcnn_transpose16(ptr(x), rows, cols, ptr(out), stream()))
    return out


def half_to_float(x: torch.Tensor, scale: float) -> torch.Tensor:
    """pcnn_half_to_float: scale * x in f32, x fp16 of any shape (contiguous)."""
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    check(lib().pcnn_half_to_float(ptr(x), x.numel(), scale, ptr(out), stream()))
    return out


def domain_tail(h9: torch.Tensor, w10: torch.Tensor, b10: torch.Tensor, label_domain: torch.Tensor | None = None,
                loss_scale: float = 1.0, grad_scale: float = 1.0) -> dict:
    """The domain classifier after fc9 (vgg16_convs.py:209-212) in one launch (pcnn_domain_tail).  h9 [rows, ld] fp16 = fc9's
    output, w10 [2][256] f32 (domain_score weights, output-major), b10 [2] f32.  Returns domain_score (after its ReLU) /
    domain_prob [rows, 2] f32 and domain_label [rows] int32; with label_domain [rows] int32 also loss [1] (loss_scale *
    sum of the rows' cross entropies), amax [1] (max |d fc9 pre-activation|), dw10 [2][256], db10 [2], db9 [256] and dpre9
    [rows, ld] fp16 = grad_scale * d fc9 pre-activation.  No host synchronisation."""
    assert h9.is_cuda and h9.dtype == torch.float16 and h9.is_contiguous() and h9.dim() == 2
    assert w10.dtype == torch.float32 and w10.is_contiguous() and w10.shape == (2, 256) and b10.dtype == torch.float32
    rows, ld = h9.shape
    dev = h9.device
    out = dict(domain_score=torch.empty((rows, 2), dtype=torch.float32, device=dev),
               domain_prob=torch.empty((rows, 2), dtype=torch.float32, device=dev),
               domain_label=torch.empty((rows,), dtype=torch.int32, device=dev))
    if label_domain is not None:
        assert label_domain.dtype == torch.int32 and label_domain.is_contiguous() and label_domain.numel() == rows
        out.update(loss=torch.empty((1,), dtype=torch.float32, device=dev), amax=torch.empty((1,), dtype=torch.float32, device=dev),
                   dw10=torch.empty((2, 256), dtype=torch.float32, device=dev), db10=torch.empty((2,), dtype=torch.float32, device=dev),
                   db9=torch.empty((256,), dtype=torch.float32, device=dev), dpre9=torch.empty((rows, ld), dtype=torch.float16, device=dev))
    g = lambda k: ptr(out.get(k))
    check(lib().pcnn_domain_tail(ptr(h9), rows, ld, ptr(w10), ptr(b10), ptr(label_domain), loss_scale, grad_scale,
                                 g("domain_score"), g("domain_prob"), g("domain_label"), g("loss"), g("amax"), g("dw10"), g("db10"),
                                 g("db9"), g("dpre9"), stream()))
    return out


def domain_grad_merge(a: torch.Tensor, scale_a: float, b: torch.Tensor, scale_b: float, shape) -> torch.Tensor:
    """f32 tensor of `shape` = scale_a * a + scale_b * b (pcnn_domain_grad_merge): the pool_score gradient of the pose head
    (a, scale_a = 1 / S) and of the domain branch (b, scale_b = -lambda / S_d, the gradient reversal), a and b fp16."""
    assert a.dtype == b.dtype == torch.float16 and a.is_contiguous() and b.is_contiguous() and a.numel() == b.numel()
    out = torch.empty(shape, dtype=torch.float32, device=a.device)
    assert out.numel() == a.numel()
    check(lib().pcnn_domain_grad_merge(ptr(a), scale_a, ptr(b), scale_b, a.numel(), ptr(out), stream()))
    return out
