"""Pose estimation from predicted object coordinates and depth on the device (csrc/coord_pose.cu, DESIGN.md §13).

`estimate_poses_3d` is the batched, CUDA-graph-capturable form: every (image, class) slot gets a pose, zero where none was found,
and nothing is copied to the host.  `CoordPoseEstimator.estimate_poses_3d` keeps the signature of the reference's
`Synthesizer.estimate_poses_3d` (lib/synthesize/synthesizer.pyx:86-94) for a lib/fcn/test.py-style caller: numpy in, the
[3,4,C] pose table written in place.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from ._lib import check, lib, ptr, require_cuda, stream, workspace

NUM_HYPOTHESES = 256
NUM_ROUNDS = 8
INFO_FIELDS = ("pixels", "hypotheses", "inliers", "energy", "exhausted", "survivor")


def estimate_poses_3d(label, depth, meta_data, extents, keys, vertex=None, lowres=None, bias_vertex=None, factor_depth=10000.0,
                      trace=False):
    """label [B,H,W] int32, depth [B,H,W] f32 raw sensor units (0 = hole), meta_data [B,...] f32 (fx, px, fy, py at 0, 2, 4, 5),
    extents [C,3] f32, keys [B] int64 (the per-image Philox keys, bit pattern of a u64); object coordinates scaled into [0,1]
    from `vertex` [B,H,W,3C] f32, or from `lowres` [B,H/8,W/8,4C] + `bias_vertex` [3C] evaluated at the sampled pixels only.
    Returns {"poses": [B,C,3,4], "info": [B,C,6]} (+ "trace_hyp": [B,256,13], "trace_round": [B,C,8,4] int32 with trace=True);
    info = INFO_FIELDS."""
    lab = require_cuda("label", label, torch.int32, 3)
    dep = require_cuda("depth", depth, torch.float32, 3)
    B, H, W = lab.shape
    if tuple(dep.shape) != (B, H, W):
        raise ValueError("depth must be [B,H,W] like label")
    meta = require_cuda("meta_data", meta_data, torch.float32).reshape(B, -1)
    ext = require_cuda("extents", extents, torch.float32, 2)
    C = ext.shape[0]
    if ext.shape[1] != 3:
        raise ValueError("extents must be [C,3]")
    k = require_cuda("keys", keys, torch.int64, 1)
    if k.shape[0] != B:
        raise ValueError("keys must be [B]")
    if vertex is not None:
        v = require_cuda("vertex", vertex, torch.float32, 4)
        if tuple(v.shape) != (B, H, W, 3 * C):
            raise ValueError("vertex must be [B,H,W,3C]")
        lr = bv = None
    else:
        if lowres is None or bias_vertex is None:
            raise ValueError("pass vertex, or lowres and bias_vertex")
        v = None
        lr = require_cuda("lowres", lowres, torch.float32, 4)
        if tuple(lr.shape) != (B, H // 8, W // 8, 4 * C):
            raise ValueError("lowres must be [B,H/8,W/8,4C]")
        bv = require_cuda("bias_vertex", bias_vertex, torch.float32).reshape(-1)
        if bv.numel() != 3 * C:
            raise ValueError("bias_vertex must have 3C values")
    dev = lab.device
    poses = torch.empty((B, C, 3, 4), dtype=torch.float32, device=dev)
    info = torch.empty((B, C, len(INFO_FIELDS)), dtype=torch.float32, device=dev)
    th = torch.empty((B, NUM_HYPOTHESES, 5 + NUM_ROUNDS), dtype=torch.int32, device=dev) if trace else None
    tr = torch.empty((B, C, NUM_ROUNDS, 4), dtype=torch.int32, device=dev) if trace else None
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_coord_pose3d_workspace_bytes(B, H, W, C, ctypes.byref(nbytes)))
    ws = workspace("coord_pose3d", nbytes.value, dev)
    check(lib().pcnn_coord_pose3d_fwd(ptr(lab), ptr(v), ptr(lr), ptr(bv), ptr(dep), ptr(meta), meta.shape[1], ptr(ext), ptr(k), B, H, W, C,
                                      factor_depth, ptr(poses), ptr(info), ptr(th), ptr(tr), ptr(ws), ws.numel(), stream()))
    out = {"poses": poses, "info": info}
    if trace:
        out["trace_hyp"], out["trace_round"] = th, tr
    return out


def assemble_records(poses, extents, meta_data, im_scale=1.0, batch_offset=0):
    """The detection records of lib/fcn/test.py:1383-1399 on the device: poses [B,C,3,4] (estimate_poses_3d), extents [C,3],
    meta_data [B,...] holding K * im_scale.  Returns (rois [B*(C-1),6] = (image + batch_offset, class, _get_bb2D(extent, pose, K) *
    im_scale), poses [B*(C-1),7] = (mat2quat(R), t), num_rows [1] int32): one row per (image, class >= 1) with t_z > 0 in
    (image, class) order, zero rows after them."""
    p = require_cuda("poses", poses, torch.float32, 4)
    B, C = p.shape[0], p.shape[1]
    if tuple(p.shape[2:]) != (3, 4):
        raise ValueError("poses must be [B,C,3,4]")
    ext = require_cuda("extents", extents, torch.float32, 2)
    meta = require_cuda("meta_data", meta_data, torch.float32).reshape(B, -1)
    dev = p.device
    rois = torch.empty((B * (C - 1), 6), dtype=torch.float32, device=dev)
    out = torch.empty((B * (C - 1), 7), dtype=torch.float32, device=dev)
    num = torch.empty((1,), dtype=torch.int32, device=dev)
    check(lib().pcnn_coord_pose3d_records(ptr(p), ptr(ext), ptr(meta), meta.shape[1], B, C, int(batch_offset), im_scale, ptr(rois),
                                          ptr(out), ptr(num), stream()))
    return rois, out, num


class CoordPoseEstimator:
    """The estimator with the reference synthesizer's calling convention (lib/fcn/test.py:1353-1401)."""

    def __init__(self, device="cuda", key=0):
        """key: the Philox key of every call (the reference draws from an unseeded per-thread generator instead)."""
        self.device = torch.device(device)
        self.key = int(key)

    def estimate_poses_3d(self, labels, depth, vertmap, extents, poses, num_classes, fx, fy, px, py, factor):
        """labels [H,W] int, depth [H,W] uint16 or float (raw sensor units), vertmap [H,W,3C] (object coordinates scaled by the
        extents), extents [C,3], poses [3,4,C] float32: written in place (zero where no pose was found)."""
        lab = np.asarray(labels)
        H, W = lab.shape[-2:]
        C = int(num_classes)
        meta = np.zeros((1, 48), np.float32)
        meta[0, :9] = (fx, 0.0, px, 0.0, fy, py, 0.0, 0.0, 1.0)
        T = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a, dtype=dt), device=self.device)
        out = estimate_poses_3d(T(lab.reshape(1, H, W), np.int32), T(np.asarray(depth).reshape(1, H, W), np.float32), T(meta, np.float32),
                                T(np.asarray(extents).reshape(C, 3), np.float32),
                                torch.tensor([self.key], dtype=torch.int64, device=self.device),
                                vertex=T(np.asarray(vertmap).reshape(1, H, W, 3 * C), np.float32), factor_depth=float(factor))
        poses[...] = out["poses"][0].permute(1, 2, 0).cpu().numpy()
