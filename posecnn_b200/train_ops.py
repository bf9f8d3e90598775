"""Training-side target generation and the training step's fused losses on the device (SURVEY.md §8(f) rank 3).

Targets follow the reference's `_generate_vertex_targets` (lib/gt_synthesize_layer/minibatch.py:543-602); `loss_cls` is
`loss_cross_entropy_single_frame` on the Hardlabel mask (lib/fcn/train.py:455-465, network.py:340) and `loss_vertex` is
`smooth_l1_loss_vertex` (lib/fcn/train.py:564-573), each the launch Trainer.forward runs.  All tensors are CUDA torch tensors;
no host synchronisation.
"""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, lib, ptr, require_cuda, stream, workspace

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
    check(lib().pcnn_vertex_targets_fwd(ptr(lab), ptr(cen), B, H, W, C, w_inside, ptr(targets), ptr(weights), stream()))
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
    check(lib().pcnn_vertex_targets_3d_fwd(ptr(lab), ptr(vm), ptr(cen), ptr(ext), B, H, W, C, w_inside, ptr(targets), ptr(weights),
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
    check(lib().pcnn_vertex_targets_instances_fwd(ptr(lab), ptr(msk), ptr(ins), B, H, W, C, ins.shape[1], w_inside, ptr(targets),
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
    check(lib().pcnn_pack_pose_meta_fwd(ptr(po), ptr(cl), ptr(kk), B, I, im_scale, int(bool(flip_x)), ptr(blob), ptr(nrows), ptr(meta),
                                        stream()))
    return blob, nrows, meta


def loss_cls(score, prob, gt_label, threshold):
    """The training step's loss_cls: loss_cross_entropy_single_frame (lib/fcn/train.py:455-465) of log_softmax(score) over the
    pixels Hardlabel(prob, gt_label, threshold) selects (network.py:340), from the raw score [B,H,W,C]; neither the log-softmax
    nor the mask is materialised.  prob [B,H,W,C] f32, gt_label [B,H,W] int32.  Returns the [2] buffer (loss, count) that the
    backward pass reads."""
    sc = require_cuda("score", score, torch.float32, 4)
    pr = require_cuda("prob", prob, torch.float32, 4)
    gt = require_cuda("gt_label", gt_label, torch.int32, 3)
    B, H, W, C = sc.shape
    if pr.shape != sc.shape or tuple(gt.shape) != (B, H, W):
        raise ValueError("prob must match score [B,H,W,C] and gt_label must be [B,H,W]")
    out = torch.empty((2,), dtype=torch.float32, device=sc.device)
    ws = _workspace(sc.device)
    check(lib().pcnn_loss_cls_hard_raw_fwd(ptr(sc), ptr(pr), ptr(gt), B, H, W, C, threshold, ptr(out), ptr(ws), ws.numel(), stream()))
    return out


def loss_vertex(lowres, bias_vertex, im_label, centers, w_inside, sigma=1.0, vertmap=None, extents=None):
    """The training step's loss_vertex: smooth_l1_loss_vertex (lib/fcn/train.py:564-573) of vertex_pred against the targets of
    generate_vertex_targets(im_label, centers, w_inside), or with vertmap [B,H,W,3] and extents [C,3] given, of
    generate_vertex_targets_3d(im_label, vertmap, centers, extents, w_inside); the targets and weights are never built.  The
    vertex values come from the 1/8-resolution head tensor lowres [B,H/8,W/8,4C] + bias_vertex [3C] (bit-identical to the dense
    vertex_pred that pcnn_up8_heads writes from them).  Returns the [2] buffer (loss, sum of weights) that the backward pass reads."""
    lab = require_cuda("im_label", im_label, torch.int32, 3)
    cen = require_cuda("centers", centers, torch.float32, 3)
    lr = require_cuda("lowres", lowres, torch.float32, 4)
    bv = require_cuda("bias_vertex", bias_vertex, torch.float32, 1)
    B, H, W = lab.shape
    C = cen.shape[1]
    if cen.shape[0] != B or cen.shape[2] != 3 or tuple(lr.shape) != (B, H // 8, W // 8, 4 * C) or bv.numel() != 3 * C:
        raise ValueError("lowres must be [B,H/8,W/8,4C] with a [3C] bias, and centers [B,C,3]")
    out = torch.empty((2,), dtype=torch.float32, device=lr.device)
    ws = _workspace(lr.device)
    vm = ext = None
    if vertmap is not None:
        lab, vm, cen, ext = _coord_inputs(lab, vertmap, cen, extents)
    check(lib().pcnn_vertex_loss_fwd(ptr(lr), ptr(bv), ptr(lab), ptr(cen), ptr(vm), ptr(ext), B, H, W, C, w_inside, sigma, ptr(out), ptr(ws),
                                     ws.numel(), stream()))
    return out
