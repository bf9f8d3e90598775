"""Hardlabel / HardlabelGrad — drop-in for lib/hard_label_layer/hard_label_op.py.

Registration: hard_label_op.cc:30-44.  Call site lib/networks/network.py:340:
hard_label(prob [B,H,W,C], gt_label [B,H,W] int32, threshold) -> [B,H,W,C] one-hot mask
(GPU semantics, hard_label_op_gpu.cu.cc:16-29).
"""
from __future__ import annotations

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream
except ImportError:
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream


def hard_label(bottom_prob, bottom_gt, threshold, name=None):
    prob = require_cuda("bottom_prob", bottom_prob, torch.float32, 4)  # hard_label_op.cc:155-156
    gt = require_cuda("bottom_gt", bottom_gt, torch.int32, 3)          # hard_label_op.cc:158-159
    B, H, W, C = prob.shape
    if tuple(gt.shape) != (B, H, W):
        raise ValueError("bottom_gt must be [B,H,W] matching bottom_prob")
    top = torch.empty_like(prob)
    check(lib().pcnn_hard_label_fwd(ptr(prob), ptr(gt), B, H, W, C, threshold, ptr(top), stream()))
    return top


def hard_label_grad(bottom_prob, bottom_gt, grad, threshold=None, name=None):
    """HardlabelGrad: zeros for prob [B,H,W,C] and gt [B,H,W] (hard_label_op_gpu.cu.cc:54-63)."""
    prob = require_cuda("bottom_prob", bottom_prob, torch.float32, 4)
    B, H, W, C = prob.shape
    g_prob = torch.empty_like(prob)
    g_gt = torch.empty((B, H, W), dtype=torch.float32, device=prob.device)
    check(lib().pcnn_hard_label_bwd(B, H, W, C, ptr(g_prob), ptr(g_gt), stream()))
    return g_prob, g_gt
