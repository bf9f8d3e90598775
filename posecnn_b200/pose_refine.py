"""Pose refinement with depth on the device (csrc/pose_refine.cu, DESIGN.md §12).

`refine_poses` is the batched, CUDA-graph-capturable form the network uses: capacity-shaped ROI / pose rows in, capacity-shaped
refined rows out, the row count stays on the device.  `Refiner.icp_python` keeps the signature of the reference's
`Synthesizer.icp_python` (lib/synthesize/synthesize.cpp:2031-2033) for a lib/fcn/test.py-style caller: numpy in, `outputs` /
`outputs_icp` written in place.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from ._lib import check, lib, ptr, require_cuda, stream, workspace
from .utils.results import ICP_ERROR_THRESHOLD, ZFAR, ZNEAR

NUM_HYPOTHESES = 8
MAX_POINTS = 4096


def refine_poses(label, depth, meta_data, rois, poses, points, num_rows=None, factor_depth=10000.0, znear=ZNEAR, zfar=ZFAR,
                 max_error=ICP_ERROR_THRESHOLD, min_pixels=400, iterations=8, batch_offset=0, trace=False):
    """label [B,H,W] int32, depth [B,H,W] f32 raw sensor units, meta_data [B,...] f32 (the 48-float records), rois / poses
    [cap,7] f32, points [C,P,3] f32 (class numbering of the label map), num_rows: device int32 [1] or None (= cap).
    Returns {"poses_refined": [cap,7], "poses_icp": [cap,7], "icp_info": [cap,4]} (+ "icp_trace": [cap,8,iterations+1,8] with
    trace=True).  Rows that are not refined are zero; icp_info = (class pixels, hypothesis, score, inliers)."""
    lab = require_cuda("label", label, torch.int32, 3)
    dep = require_cuda("depth", depth, torch.float32, 3)
    B, H, W = lab.shape
    if tuple(dep.shape) != (B, H, W):
        raise ValueError("depth must be [B,H,W] like label")
    meta = require_cuda("meta_data", meta_data, torch.float32).reshape(B, -1)
    r = require_cuda("rois", rois, torch.float32, 2)
    p = require_cuda("poses", poses, torch.float32, 2)
    cap = r.shape[0]
    if r.shape[1] != 7 or tuple(p.shape) != (cap, 7):
        raise ValueError("rois and poses must be [cap,7]")
    pts = require_cuda("points", points, torch.float32, 3)
    C, P = pts.shape[0], pts.shape[1]
    if pts.shape[2] != 3:
        raise ValueError("points must be [C,P,3]")
    nr = None if num_rows is None else require_cuda("num_rows", num_rows, torch.int32).reshape(-1)
    dev = lab.device
    out_r = torch.empty((cap, 7), dtype=torch.float32, device=dev)
    out_i = torch.empty((cap, 7), dtype=torch.float32, device=dev)
    info = torch.empty((cap, 4), dtype=torch.float32, device=dev)
    tr = torch.empty((cap, NUM_HYPOTHESES, max(int(iterations), 0) + 1, 8), dtype=torch.float32, device=dev) if trace else None
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_pose_refine_workspace_bytes(B, max(C, 2), ctypes.byref(nbytes)))
    ws = workspace("pose_refine", nbytes.value, dev)
    check(lib().pcnn_pose_refine_fwd(ptr(lab), ptr(dep), ptr(meta), meta.shape[1], ptr(r), ptr(p), ptr(nr), cap, ptr(pts), C, P, B, H, W,
                                     int(batch_offset), factor_depth, znear, zfar, max_error, int(min_pixels), int(iterations), ptr(out_r),
                                     ptr(out_i), ptr(info), ptr(tr), ptr(ws), ws.numel(), stream()))
    out = {"poses_refined": out_r, "poses_icp": out_i, "icp_info": info}
    if tr is not None:
        out["icp_trace"] = tr
    return out


class Refiner:
    """The refiner with the reference synthesizer's calling convention (lib/fcn/test.py:1327-1351)."""

    def __init__(self, points, device="cuda"):
        """points [C,P,3]: the model point table in the label map's class numbering (imdb._points_all)."""
        self.points = torch.as_tensor(np.asarray(points, dtype=np.float32), device=device).contiguous()
        self.device = self.points.device

    def icp_python(self, labelmap, depth, parameters, height, width, num_roi, channel_roi, rois, poses, outputs, outputs_icp, maxError):
        """labelmap [H,W] int, depth [H,W] uint16 or float (raw sensor units), parameters = results.icp_parameters (fx, fy, px, py,
        znear, zfar, factor), rois [num_roi, channel_roi] (class in column 1; the batch column is ignored, as the reference does),
        poses [num_roi,7].  Writes outputs (poses_refined) and outputs_icp (poses_icp) [num_roi,7] in place."""
        H, W, n = int(height), int(width), int(num_roi)
        if n == 0:
            return
        prm = np.asarray(parameters, dtype=np.float64).reshape(-1)
        fx, fy, px, py, znear, zfar, factor = (float(v) for v in prm[:7])
        meta = np.zeros((1, 48), np.float32)
        meta[0, :9] = (fx, 0.0, px, 0.0, fy, py, 0.0, 0.0, 1.0)
        r = np.zeros((n, 7), np.float32)
        r[:, 1] = np.asarray(rois, np.float32).reshape(n, int(channel_roi))[:, 1]
        T = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a, dtype=dt), device=self.device)
        out = refine_poses(T(np.asarray(labelmap).reshape(1, H, W), np.int32), T(np.asarray(depth).reshape(1, H, W), np.float32),
                           T(meta, np.float32), T(r, np.float32), T(np.asarray(poses).reshape(n, 7), np.float32), self.points,
                           factor_depth=factor, znear=znear, zfar=zfar, max_error=float(maxError))
        outputs[:n] = out["poses_refined"].cpu().numpy()
        outputs_icp[:n] = out["poses_icp"].cpu().numpy()
