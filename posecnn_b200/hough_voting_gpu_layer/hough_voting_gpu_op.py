"""Houghvotinggpu — drop-in for lib/hough_voting_gpu_layer/hough_voting_gpu_op.py.

Reference registration: hough_voting_gpu_op.cc:37-52 (inputs bottom_label:int32,
bottom_vertex, bottom_extents, bottom_meta_data, bottom_gt; attrs is_train,
threshold_vote, threshold_percentage, skip_pixels; outputs top_box, top_pose,
top_target, top_weight, top_domain:int32).  Call site: lib/networks/network.py:258-259.
Tensors are CUDA torch tensors in the reference's NHWC layouts.
"""
from __future__ import annotations

import ctypes

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream, workspace
except ImportError:  # posecnn_b200/ itself on sys.path (reference-style imports)
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream, workspace

MAX_ROWS = 128 * 9          # hough_voting_gpu_op.cc:94
INLIER_THRESHOLD = 0.9      # hough_voting_gpu_op.cc:356
LABEL_THRESHOLD = 500       # hough_voting_gpu_op.cc:357


def hough_voting_gpu_capacity(bottom_label, bottom_vertex, bottom_extents, bottom_meta_data, bottom_gt, is_train,
                              threshold_vote, threshold_percentage, skip_pixels,
                              inlier_threshold=INLIER_THRESHOLD, label_threshold=LABEL_THRESHOLD,
                              lowres=None, bias_vertex=None, batch_global=None, batch_offset=0):
    """Stream-ordered form: returns the five 1152-row capacity buffers, the device row
    count [1] int32 and a device status word; no host synchronisation.

    Pipeline extensions (pcnn_hough_vote_fwd_ex): `bottom_vertex=None` + `lowres` [B,H/8,W/8,4C] + `bias_vertex` [3C]
    samples the vertex head on demand instead of reading a dense vertex_pred (bit-identical); `batch_global` /
    `batch_offset` make this call one image shard of a larger batch (ROI cap 128 // batch_global, global batch indices)."""
    label = require_cuda("bottom_label", bottom_label, torch.int32, 3)       # .cc:328-329
    extents = require_cuda("bottom_extents", bottom_extents, torch.float32)
    meta = require_cuda("bottom_meta_data", bottom_meta_data, torch.float32)
    B, H, W = label.shape
    if bottom_vertex is not None:
        vertex = require_cuda("bottom_vertex", bottom_vertex, torch.float32, 4)  # .cc:331-332
        if vertex.shape[0] != B or vertex.shape[1] != H or vertex.shape[2] != W or vertex.shape[3] % 3:
            raise ValueError("bottom_vertex must be [B,H,W,3*num_classes] matching bottom_label")
        C = vertex.shape[3] // 3
        lowres = bias_vertex = None
    else:
        vertex = None
        lowres = require_cuda("lowres", lowres, torch.float32, 4)
        bias_vertex = require_cuda("bias_vertex", bias_vertex, torch.float32, 1)
        if lowres.shape[0] != B or lowres.shape[1] * 8 != H or lowres.shape[2] * 8 != W or lowres.shape[3] % 4:
            raise ValueError("lowres must be [B,H/8,W/8,4*num_classes] matching bottom_label")
        C = lowres.shape[3] // 4
        if bias_vertex.numel() != 3 * C:
            raise ValueError("bias_vertex must be [3*num_classes]")
    if extents.numel() != C * 3:
        raise ValueError("bottom_extents must be [num_classes,3]")
    num_meta = meta.shape[-1]
    if meta.numel() != B * num_meta:
        raise ValueError("bottom_meta_data must hold one record per image")
    if bottom_gt is None or bottom_gt.numel() == 0:
        gt, num_gt = None, 0
    else:
        gt = require_cuda("bottom_gt", bottom_gt, torch.float32).reshape(-1, 13)
        num_gt = gt.shape[0]
    bg = B if batch_global is None else int(batch_global)
    dev = label.device
    box = torch.empty((MAX_ROWS, 7), dtype=torch.float32, device=dev)
    pose = torch.empty((MAX_ROWS, 7), dtype=torch.float32, device=dev)
    target = torch.empty((MAX_ROWS, 4 * C), dtype=torch.float32, device=dev)
    weight = torch.empty((MAX_ROWS, 4 * C), dtype=torch.float32, device=dev)
    domain = torch.empty((MAX_ROWS,), dtype=torch.int32, device=dev)
    num_rois = torch.empty((1,), dtype=torch.int32, device=dev)
    status = torch.empty((4,), dtype=torch.int32, device=dev)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_hough_vote_workspace_bytes(B, H, W, C, int(skip_pixels), threshold_vote, ctypes.byref(nbytes)))
    ws = workspace("hough", nbytes.value, dev)
    check(lib().pcnn_hough_vote_fwd_ex(ptr(label), ptr(vertex), ptr(lowres), ptr(bias_vertex), ptr(extents), ptr(meta), ptr(gt), B, bg,
                                       int(batch_offset), H, W, C, num_gt, num_meta, int(is_train), inlier_threshold, int(label_threshold),
                                       threshold_vote, threshold_percentage, int(skip_pixels), ptr(box), ptr(pose), ptr(target),
                                       ptr(weight), ptr(domain), ptr(num_rois), ptr(status), ptr(ws), ws.numel(), stream()))
    return box, pose, target, weight, domain, num_rois, status


def check_status(overflow_bits: int, mismatches: int):
    """The device status word of pcnn_hough_vote_fwd (include/posecnn_b200.h): bit 0 of [0] = the per-image candidate
    list of threshold mode overflowed (which maxima survive then depends on atomic arrival order, like the reference's
    own `atomicAdd` compaction, .cu.cc:377 — the canonical order is lost); [1] = selected cells whose interval-scan
    vote differs from the exact per-cell recount (the reported vote is always the recount)."""
    import warnings
    if overflow_bits & 1:
        warnings.warn("Houghvotinggpu: more local maxima than the candidate capacity (4096 per image); the kept subset is "
                      "not in canonical order", RuntimeWarning)
    if mismatches:
        warnings.warn("Houghvotinggpu: %d selected cells sit within rounding distance of the vote predicate's threshold "
                      "(interval scan != per-cell recount; the recount is reported)" % mismatches, RuntimeWarning)


def hough_voting_gpu(bottom_label, bottom_vertex, bottom_extents, bottom_meta_data, bottom_gt, is_train,
                     threshold_vote, threshold_percentage, skip_pixels, name=None):
    """Same positional order as the TF op.  Output row count is data dependent and always
    >= 1 (dummy all-zero row, hough_voting_gpu_op.cc:379-383), hence one host read of the
    device row counter, as in the reference (copy_num_rois, .cu.cc:591-594)."""
    box, pose, target, weight, domain, num_rois, status = hough_voting_gpu_capacity(
        bottom_label, bottom_vertex, bottom_extents, bottom_meta_data, bottom_gt, is_train, threshold_vote,
        threshold_percentage, skip_pixels)
    host = torch.cat([num_rois, status[:2]]).tolist()     # the one host read the data-dependent shape requires
    n = max(1, host[0])
    check_status(host[1], host[2])
    return box[:n], pose[:n], target[:n], weight[:n], domain[:n]


def hough_voting_gpu_grad(bottom_label, bottom_vertex, grad, name=None):
    """HoughvotinggpuGrad (hough_voting_gpu_op.cc:54-60; set_gradients .cu.cc:608-612): zeros."""
    label = require_cuda("bottom_label", bottom_label, torch.int32, 3)
    vertex = require_cuda("bottom_vertex", bottom_vertex, torch.float32, 4)
    B, H, W = label.shape
    C = vertex.shape[3] // 3
    g_label = torch.empty((B, H, W), dtype=torch.float32, device=label.device)
    g_vertex = torch.empty_like(vertex)
    check(lib().pcnn_hough_vote_bwd(ptr(g_label), ptr(g_vertex), B, H, W, C, stream()))
    return g_label, g_vertex


def hough_vote_planes(bottom_label, bottom_vertex, bottom_extents, bottom_meta_data, skip_pixels,
                      inlier_threshold=INLIER_THRESHOLD, label_threshold=LABEL_THRESHOLD):
    """Dense vote planes [B,C,H,W] from the same kernels (parity/debug helper)."""
    label = require_cuda("bottom_label", bottom_label, torch.int32, 3)
    vertex = require_cuda("bottom_vertex", bottom_vertex, torch.float32, 4)
    extents = require_cuda("bottom_extents", bottom_extents, torch.float32)
    meta = require_cuda("bottom_meta_data", bottom_meta_data, torch.float32)
    B, H, W = label.shape
    C = vertex.shape[3] // 3
    votes = torch.empty((B, C, H, W), dtype=torch.float32, device=label.device)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_hough_vote_workspace_bytes(B, H, W, C, int(skip_pixels), -1.0, ctypes.byref(nbytes)))
    ws = workspace("hough", nbytes.value, label.device)
    check(lib().pcnn_hough_vote_planes(ptr(label), ptr(vertex), ptr(extents), ptr(meta), B, H, W, C, meta.shape[-1], inlier_threshold,
                                       int(label_threshold), int(skip_pixels), ptr(votes), ptr(ws), ws.numel(), stream()))
    return votes
