"""Training-side target generation and fused losses on the device (SURVEY.md §8(f) rank 3).

Names follow the reference: `_generate_vertex_targets` (lib/gt_synthesize_layer/minibatch.py:543-602),
`loss_cross_entropy_single_frame` on the Hardlabel mask (lib/fcn/train.py:455-465, network.py:340) and
`smooth_l1_loss_vertex` (lib/fcn/train.py:564-573).  All tensors are CUDA torch tensors; no host synchronisation.
"""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, f32, lib, ptr, require_cuda, stream, workspace

def _workspace(device):
    n = ctypes.c_size_t(0)
    check(lib().pcnn_train_loss_workspace_bytes(ctypes.byref(n)))
    return workspace("train_loss", int(n.value), device, zero=True)   # zero once: the kernels re-arm the ticket


def generate_vertex_targets(im_label, centers, w_inside=1.0):
    """im_label [B,H,W] int32; centers [B,C,3] f32 = (cx, cy, z) per class, z <= 0 where the class is not in the image
    (center[ind] / poses[2,3,ind] of minibatch.py:585-587).  Returns (vertex_targets, vertex_weights) [B,H,W,3C] f32."""
    lab = require_cuda("im_label", im_label, torch.int32, 3)
    cen = require_cuda("centers", centers, torch.float32, 3)
    B, H, W = lab.shape
    C = cen.shape[1]
    if cen.shape[0] != B or cen.shape[2] != 3:
        raise ValueError("centers must be [B,C,3]")
    targets = torch.empty((B, H, W, 3 * C), dtype=torch.float32, device=lab.device)
    weights = torch.empty_like(targets)
    check(lib().pcnn_vertex_targets_fwd(ptr(lab), ptr(cen), B, H, W, C, f32(w_inside), ptr(targets), ptr(weights), stream()))
    return targets, weights


def _coord_inputs(im_label, vertmap, centers, extents):
    lab = require_cuda("im_label", im_label, torch.int32, 3)
    vm = require_cuda("vertmap", vertmap, torch.float32, 4)
    cen = require_cuda("centers", centers, torch.float32, 3)
    ext = require_cuda("extents", extents, torch.float32, 2)
    B, H, W = lab.shape
    C = cen.shape[1]
    if tuple(vm.shape) != (B, H, W, 3) or cen.shape[0] != B or cen.shape[2] != 3 or tuple(ext.shape) != (C, 3):
        raise ValueError("vertmap must be [B,H,W,3], centers [B,C,3] and extents [C,3]")
    return lab, vm, cen, ext


def generate_vertex_targets_3d(im_label, vertmap, centers, extents, w_inside=1.0):
    """The VERTEX_REG_3D branch of _generate_vertex_targets (minibatch.py:595-600, _scale_vertmap :605-616): im_label [B,H,W] int32,
    vertmap [B,H,W,3] f32 (each pixel's object coordinate, metres in the model frame), centers [B,C,3] f32 (only z > 0 is read: the
    class is listed in the frame), extents [C,3] f32.  A pixel of a listed class c in 1..C-1 gets (vertmap - vmin) / (vmax - vmin)
    per axis in channels 3c..3c+2 (the reference's float32 a * v + b) and weight w_inside there.  Returns (vertex_targets,
    vertex_weights) [B,H,W,3C] f32."""
    lab, vm, cen, ext = _coord_inputs(im_label, vertmap, centers, extents)
    B, H, W = lab.shape
    C = cen.shape[1]
    targets = torch.empty((B, H, W, 3 * C), dtype=torch.float32, device=lab.device)
    weights = torch.empty_like(targets)
    check(lib().pcnn_vertex_targets_3d_fwd(ptr(lab), ptr(vm), ptr(cen), ptr(ext), B, H, W, C, f32(w_inside), ptr(targets), ptr(weights),
                                           stream()))
    return targets, weights


def generate_vertex_targets_instances(im_label, mask, instances, num_classes, w_inside=1.0):
    """Multi-instance branch of _generate_vertex_targets (minibatch.py:549-573): im_label / mask [B,H,W] int32 (instance
    mask image), instances [B,I,5] f32 = (cls, mask id = cls_indexes_old + 1, cx, cy, z), z <= 0 = unused slot."""
    lab = require_cuda("im_label", im_label, torch.int32, 3)
    msk = require_cuda("mask", mask, torch.int32, 3)
    ins = require_cuda("instances", instances, torch.float32, 3)
    B, H, W = lab.shape
    if msk.shape != lab.shape or ins.shape[0] != B or ins.shape[2] != 5:
        raise ValueError("mask must match im_label and instances must be [B,I,5]")
    C = int(num_classes)
    targets = torch.empty((B, H, W, 3 * C), dtype=torch.float32, device=lab.device)
    weights = torch.empty_like(targets)
    check(lib().pcnn_vertex_targets_instances_fwd(ptr(lab), ptr(msk), ptr(ins), B, H, W, C, ins.shape[1], f32(w_inside), ptr(targets),
                                                  ptr(weights), stream()))
    return targets, weights


def pack_pose_meta(poses, cls, intrinsics, im_scale=1.0, flip_x=False):
    """The data layer's pose blob and meta_data packing on the device (minibatch.py:440-451, 474-492): poses [B,I,3,4] f32
    ([R|T] per listed instance), cls [B,I] int32 (< 0 = unused slot), intrinsics [B,3,3] f32 -> (pose_blob capacity buffer
    [B*I,13], num_rows [1] int32 on the device, meta_data [B,1,1,48])."""
    po = require_cuda("poses", poses, torch.float32, 4)
    cl = require_cuda("cls", cls, torch.int32, 2)
    kk = require_cuda("intrinsics", intrinsics, torch.float32, 3)
    B, I = cl.shape
    blob = torch.empty((B * I, 13), dtype=torch.float32, device=po.device)
    nrows = torch.empty((1,), dtype=torch.int32, device=po.device)
    meta = torch.empty((B, 1, 1, 48), dtype=torch.float32, device=po.device)
    check(lib().pcnn_pack_pose_meta_fwd(ptr(po), ptr(cl), ptr(kk), B, I, f32(im_scale), int(bool(flip_x)), ptr(blob), ptr(nrows), ptr(meta),
                                        stream()))
    return blob, nrows, meta


def loss_cross_entropy_hard(scores, prob, gt_label, threshold, want_grad=False, upstream=1.0):
    """-sum(hard_label(prob, gt, threshold) * scores) / (sum(mask) + 1e-10) with scores = log-softmax [B,H,W,C];
    the mask is never materialised.  Returns (loss [1] view, count [1] view[, grad wrt scores])."""
    sc = require_cuda("scores", scores, torch.float32, 4)
    pr = require_cuda("prob", prob, torch.float32, 4)
    gt = require_cuda("gt_label", gt_label, torch.int32, 3)
    B, H, W, C = sc.shape
    out = torch.empty((2,), dtype=torch.float32, device=sc.device)
    grad = torch.empty_like(sc) if want_grad else None
    ws = _workspace(sc.device)
    check(lib().pcnn_loss_cls_hard_fwd(ptr(sc), ptr(pr), ptr(gt), B, H, W, C, f32(threshold), ptr(out), f32(upstream), ptr(grad),
                                       ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
    return (out[0:1], out[1:2], grad) if want_grad else (out[0:1], out[1:2])


def smooth_l1_loss_vertex(vertex_pred, vertex_targets, vertex_weights, sigma=1.0, want_grad=False, upstream=1.0):
    """lib/fcn/train.py:564-573.  Returns (loss [1], sum of weights [1][, grad wrt vertex_pred])."""
    p = require_cuda("vertex_pred", vertex_pred, torch.float32, vertex_pred.dim())
    t = require_cuda("vertex_targets", vertex_targets, torch.float32, vertex_pred.dim())
    w = require_cuda("vertex_weights", vertex_weights, torch.float32, vertex_pred.dim())
    if t.shape != p.shape or w.shape != p.shape:
        raise ValueError("vertex_pred, vertex_targets and vertex_weights must have the same shape")
    out = torch.empty((2,), dtype=torch.float32, device=p.device)
    grad = torch.empty_like(p) if want_grad else None
    ws = _workspace(p.device)
    check(lib().pcnn_smooth_l1_vertex_fwd(ptr(p), ptr(t), ptr(w), ctypes.c_size_t(p.numel()), f32(sigma), ptr(out), f32(upstream),
                                          ptr(grad), ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
    return (out[0:1], out[1:2], grad) if want_grad else (out[0:1], out[1:2])


def vertex_loss_from_centers(vertex_pred, im_label, centers, w_inside=1.0, sigma=1.0, want_grad=False, upstream=1.0):
    """smooth_l1_loss_vertex(vertex_pred, *generate_vertex_targets(im_label, centers, w_inside)) in one pass that never
    builds the target / weight tensors.  Returns (loss [1], sum of weights [1][, grad wrt vertex_pred])."""
    p = require_cuda("vertex_pred", vertex_pred, torch.float32, 4)
    lab = require_cuda("im_label", im_label, torch.int32, 3)
    cen = require_cuda("centers", centers, torch.float32, 3)
    B, H, W = lab.shape
    C = cen.shape[1]
    if tuple(p.shape) != (B, H, W, 3 * C) or cen.shape[0] != B or cen.shape[2] != 3:
        raise ValueError("vertex_pred must be [B,H,W,3C] and centers [B,C,3]")
    out = torch.empty((2,), dtype=torch.float32, device=p.device)
    grad = torch.empty_like(p) if want_grad else None
    ws = _workspace(p.device)
    check(lib().pcnn_vertex_loss_fused_fwd(ptr(p), ptr(lab), ptr(cen), B, H, W, C, f32(w_inside), f32(sigma), ptr(out), f32(upstream),
                                           ptr(grad), ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
    return (out[0:1], out[1:2], grad) if want_grad else (out[0:1], out[1:2])


def vertex_loss_from_coords(vertex_pred, im_label, vertmap, centers, extents, w_inside=1.0, sigma=1.0, want_grad=False, upstream=1.0,
                            bias_vertex=None):
    """smooth_l1_loss_vertex(vertex_pred, *generate_vertex_targets_3d(im_label, vertmap, centers, extents, w_inside)) in one pass that
    never builds the target / weight tensors.  vertex_pred is the dense [B,H,W,3C] tensor, or with bias_vertex [3C] given, the
    1/8-resolution head tensor [B,H/8,W/8,4C] whose vertex values are formed on demand (bit-identical; no gradient then).
    Returns (loss [1], sum of weights [1][, grad wrt vertex_pred])."""
    lab, vm, cen, ext = _coord_inputs(im_label, vertmap, centers, extents)
    B, H, W = lab.shape
    C = cen.shape[1]
    p = require_cuda("vertex_pred", vertex_pred, torch.float32, 4)
    out = torch.empty((2,), dtype=torch.float32, device=p.device)
    ws = _workspace(p.device)
    if bias_vertex is not None:
        if want_grad:
            raise ValueError("the low-resolution source has no gradient output")
        bv = require_cuda("bias_vertex", bias_vertex, torch.float32, 1)
        if tuple(p.shape) != (B, H // 8, W // 8, 4 * C) or bv.numel() != 3 * C:
            raise ValueError("the low-resolution source must be [B,H/8,W/8,4C] with a [3C] bias")
        check(lib().pcnn_vertex_loss_coord_lowres_fwd(ptr(p), ptr(bv), ptr(lab), ptr(vm), ptr(cen), ptr(ext), B, H, W, C, f32(w_inside),
                                                      f32(sigma), ptr(out), ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
        return out[0:1], out[1:2]
    if tuple(p.shape) != (B, H, W, 3 * C):
        raise ValueError("vertex_pred must be [B,H,W,3C]")
    grad = torch.empty_like(p) if want_grad else None
    check(lib().pcnn_vertex_loss_coord_fwd(ptr(p), ptr(lab), ptr(vm), ptr(cen), ptr(ext), B, H, W, C, f32(w_inside), f32(sigma), ptr(out),
                                           f32(upstream), ptr(grad), ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
    return (out[0:1], out[1:2], grad) if want_grad else (out[0:1], out[1:2])
