"""Region proposals on the device: lib/rpn_layer/proposal_layer.py for a batch of images (csrc/det.cu, DESIGN.md §16).

`proposal_layer` keeps the reference's argument order; its inputs carry a batch dimension and its outputs are capacity-shaped
(post_top_n rows per image, a device count per image), so no host synchronisation is needed.  `rpn_heads` is the pair of 1x1
convolutions and the pair softmax that feed it (vgg16_det.py:99-106).
"""
from __future__ import annotations

import ctypes

import torch

from .._lib import check, lib, ptr, require_cuda, stream, workspace

# (RPN_PRE_NMS_TOP_N, RPN_POST_NMS_TOP_N, RPN_NMS_THRESH) of lib/fcn/config.py:171-177 (TRAIN) and 224-231 (TEST)
CFG = {"TRAIN": (12000, 2000, 0.7), "TEST": (6000, 300, 0.7)}


def rpn_heads(conv_rpn: torch.Tensor, w_tc: torch.Tensor, bias: torch.Tensor, num_anchors: int):
    """conv_rpn [B,h,w,512] bf16, w_tc [6A,512] bf16 (rpn_cls_score's 2A output channels, then rpn_bbox_pred's 4A), bias [6A] f32
    -> rpn_cls_prob [B,h,w,2A] f32, rpn_bbox_pred [B,h,w,4A] f32 (both 1x1 convolutions with ReLU, then the pair softmax)."""
    x = require_cuda("conv_rpn", conv_rpn, torch.bfloat16, 4)
    w_tc = require_cuda("w_tc", w_tc, torch.bfloat16, 2)
    bias = require_cuda("bias", bias, torch.float32, 1)
    A = int(num_anchors)
    B, h, w, cin = x.shape
    if cin != 512 or tuple(w_tc.shape) != (6 * A, 512) or bias.numel() != 6 * A:
        raise ValueError("rpn_heads: conv_rpn [B,h,w,512], w_tc [6A,512] and bias [6A] expected")
    if w_tc.device != x.device or bias.device != x.device:
        raise ValueError("rpn_heads: conv_rpn, w_tc and bias must be on the same device")
    prob = torch.empty((B, h, w, 2 * A), dtype=torch.float32, device=x.device)
    deltas = torch.empty((B, h, w, 4 * A), dtype=torch.float32, device=x.device)
    check(lib().pcnn_rpn_heads_fwd(ptr(x), ptr(w_tc), ptr(bias), B * h * w, A, ptr(prob), ptr(deltas), stream()))
    return prob, deltas


def proposals(rpn_cls_prob, rpn_bbox_pred, anchors, im_h, im_w, pre_top_n, post_top_n, nms_thresh, want_pre_boxes=False):
    """The proposal layer with explicit settings.  rpn_cls_prob [B,h,w,2A], rpn_bbox_pred [B,h,w,4A], anchors [h*w*A,4] f32 on the
    device -> rois [B*post_top_n,5] (b, x1, y1, x2, y2), scores [B*post_top_n,1], num_rois [B] int32; with want_pre_boxes also
    the sorted, decoded and clipped candidates NMS ran on, [B,K,5] (x1, y1, x2, y2, score), K = min(pre_top_n, h*w*A)."""
    prob = require_cuda("rpn_cls_prob", rpn_cls_prob, torch.float32, 4)
    deltas = require_cuda("rpn_bbox_pred", rpn_bbox_pred, torch.float32, 4)
    anc = require_cuda("anchors", anchors, torch.float32, 2)
    B, h, w, a2 = prob.shape
    A = a2 // 2
    if a2 % 2 or tuple(deltas.shape) != (B, h, w, 4 * A) or tuple(anc.shape) != (h * w * A, 4):
        raise ValueError("proposals: rpn_cls_prob [B,h,w,2A], rpn_bbox_pred [B,h,w,4A] and anchors [h*w*A,4] expected")
    if deltas.device != prob.device or anc.device != prob.device:
        raise ValueError("proposals: rpn_cls_prob, rpn_bbox_pred and anchors must be on the same device")
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_rpn_proposals_workspace_bytes(B, h, w, A, int(pre_top_n), ctypes.byref(nbytes)))
    ws = workspace("rpn_proposals", nbytes.value, prob.device)
    post = int(post_top_n)
    dev = prob.device
    rois = torch.empty((B * post, 5), dtype=torch.float32, device=dev)
    scores = torch.empty((B * post, 1), dtype=torch.float32, device=dev)
    num = torch.empty((B,), dtype=torch.int32, device=dev)
    K = min(int(pre_top_n), h * w * A)
    pre = torch.empty((B, K, 5), dtype=torch.float32, device=dev) if want_pre_boxes else None
    check(lib().pcnn_rpn_proposals_fwd(ptr(prob), ptr(deltas), ptr(anc), B, h, w, A, float(im_h), float(im_w), int(pre_top_n), post,
                                       float(nms_thresh), ptr(rois), ptr(scores), ptr(num), ptr(pre), ptr(ws), ws.numel(), stream()))
    return (rois, scores, num, pre) if want_pre_boxes else (rois, scores, num)


def proposal_layer(rpn_cls_prob, rpn_bbox_pred, im_info, cfg_key, _feat_stride, anchors, num_anchors):
    """proposal_layer.py's signature with a batch dimension: rpn_cls_prob [B,h,w,2A], rpn_bbox_pred [B,h,w,4A], im_info (height,
    width, scale) of the blob (host numbers), cfg_key 'TEST' or 'TRAIN' (top-N and NMS threshold of lib/fcn/config.py), anchors
    [h*w*A,4] (snippets.generate_anchors_pre, on the device).  Returns rois [B*N,5] with rois[:,0] the image index, rpn_scores
    [B*N,1] and num_rois [B] int32 on the device, N = RPN_POST_NMS_TOP_N; rows past an image's count are zero boxes carrying its
    index.  _feat_stride is implied by the anchors, as in the reference."""
    if isinstance(cfg_key, bytes):
        cfg_key = cfg_key.decode("utf-8")
    if cfg_key not in CFG:
        raise ValueError(f"cfg_key must be 'TEST' or 'TRAIN', got {cfg_key!r}")
    if rpn_cls_prob.shape[-1] != 2 * int(num_anchors):
        raise ValueError(f"rpn_cls_prob has {rpn_cls_prob.shape[-1]} channels, not 2 * num_anchors = {2 * int(num_anchors)}")
    pre, post, thresh = CFG[cfg_key]
    im_h, im_w = (float(v) for v in list(im_info)[:2])
    return proposals(rpn_cls_prob, rpn_bbox_pred, anchors, im_h, im_w, pre, post, thresh)
