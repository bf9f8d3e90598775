"""Detection records on the device: the end of lib/fcn/test.py's test loop for the detection network (csrc/det.cu,
DESIGN.md §16).

`detection_records` turns the five tensors vgg16_det's forward leaves (cls_prob, bbox_pred, rois, num_rois, poses_tanh) into
one record per (image, foreground class): the top-scoring proposal of the class above 0.02 (test.py:1589-1616, whose
`nms(...)` then `keep[0]` keeps exactly that row), its class box (test.py:1731-1746) and the translation of
compute_translations (test.py:1639-1691), a Nelder-Mead fit of the projected model points to the box.  Records stay on the
device in fixed slots, so the stage needs no host synchronisation and can be captured in a CUDA graph.
"""
from __future__ import annotations

import torch

from ._lib import check, lib, ptr, require_cuda, stream


def detection_records(cls_prob, bbox_pred, poses_tanh, rois, num_rois, im_hw, meta_data, points):
    """cls_prob [B*N,C], bbox_pred [B*N,4C] (normalised deltas, as the network emits them), poses_tanh [B*N,4C], rois [B*N,5]
    (b, x1, y1, x2, y2) f32 and num_rois [B] int32 (the first num_rois[b] of image b's N rows count) on the device; im_hw
    (height, width) of the image the boxes are clipped to; meta_data [B,>=9] f32 (K = meta_data[b, 0:9]); points [C,P,3] f32,
    the object-point table (P <= 4096, class 0 unused).

    Returns dets [B*(C-1),7] (b, class, x1, y1, x2, y2, score), poses [B*(C-1),7] (qw, qx, qy, qz, tx, ty, tz), num_dets [B]
    int32 and trace [B*(C-1),2] int32 (Nelder-Mead iterations, objective evaluations).  Slot b*(C-1) + j-1 holds class j of
    image b; a class with no proposal above 0.02 leaves its slot empty: (b, 0, 0, 0, 0, 0, 0) with a zero pose, which pairs
    with no ground truth in Evaluator.add_poses."""
    P_ = require_cuda("cls_prob", cls_prob, torch.float32, 2)
    D = require_cuda("bbox_pred", bbox_pred, torch.float32, 2)
    Q = require_cuda("poses_tanh", poses_tanh, torch.float32, 2)
    R = require_cuda("rois", rois, torch.float32, 2)
    n = require_cuda("num_rois", num_rois, torch.int32, 1)
    meta = require_cuda("meta_data", meta_data, torch.float32, (2, 3))
    pts = require_cuda("points", points, torch.float32, 3)
    dev = P_.device
    if any(t.device != dev for t in (D, Q, R, n, meta, pts)):
        raise ValueError("detection_records: every tensor must be on the same device")
    B = n.shape[0]
    rows, C = P_.shape
    if B < 1 or rows % B:
        raise ValueError(f"detection_records: {rows} rows do not split into {B} images")
    if tuple(D.shape) != (rows, 4 * C) or tuple(Q.shape) != (rows, 4 * C) or tuple(R.shape) != (rows, 5):
        raise ValueError("detection_records: bbox_pred and poses_tanh [B*N,4C], rois [B*N,5] expected")
    meta = meta.reshape(meta.shape[0], -1)
    if meta.shape[0] != B or pts.shape[0] != C or pts.shape[2] != 3:
        raise ValueError("detection_records: meta_data [B,>=9] and points [C,P,3] expected")
    im_h, im_w = (int(v) for v in im_hw)
    S = B * (C - 1)
    dets = torch.empty((S, 7), dtype=torch.float32, device=dev)
    poses = torch.empty((S, 7), dtype=torch.float32, device=dev)
    num_dets = torch.empty((B,), dtype=torch.int32, device=dev)
    trace = torch.empty((S, 2), dtype=torch.int32, device=dev)
    check(lib().pcnn_det_records_fwd(ptr(P_), ptr(D), ptr(Q), ptr(R), ptr(n), B, rows // B, C, im_h, im_w, ptr(meta), meta.shape[1],
                                     ptr(pts), pts.shape[1], ptr(dets), ptr(poses), ptr(num_dets), ptr(trace), stream()))
    return dets, poses, num_dets, trace
