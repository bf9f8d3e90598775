"""Device-side NMS + pose assembly — drop-in for lib/utils/nms.py and the loop of lib/fcn/test.py:197-211.

`nms(dets, thresh)` keeps the reference's signature (dets = Hough ROI rows [batch, cls, x1, y1, x2, y2, score]) and
returns the kept row indices in processing order.  `nms_pose_capacity` is the graph-friendly form the network uses:
fixed-size outputs + a device count, no host synchronisation.
"""
from __future__ import annotations

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream
except ImportError:
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream


def nms_pose_capacity(rois, poses_init, poses_pred=None, num_rois=None, thresh=0.5, per_image=True, num_classes=None):
    """rois [cap,7] f32, poses_init [cap,7], poses_pred [cap,4C] or None, num_rois: device int32 [1] (Hough's row
    count) or None (all rows).  Returns (keep [cap] i32, rois [cap,7], poses [cap,7], num_keep [1] i32)."""
    r = require_cuda("rois", rois, torch.float32, 2)
    pi = require_cuda("poses_init", poses_init, torch.float32, 2)
    cap = r.shape[0]
    if r.shape[1] != 7 or tuple(pi.shape) != (cap, 7):
        raise ValueError("rois and poses_init must be [N,7]")
    C = 0
    pp = None
    if poses_pred is not None:
        pp = require_cuda("poses_pred", poses_pred, torch.float32, 2)
        if pp.shape[0] != cap or pp.shape[1] % 4:
            raise ValueError("poses_pred must be [N,4C]")
        C = pp.shape[1] // 4 if num_classes is None else int(num_classes)
    nr = None if num_rois is None else require_cuda("num_rois", num_rois, torch.int32, 1)
    keep = torch.empty((cap,), dtype=torch.int32, device=r.device)
    out_r = torch.empty_like(r)
    out_p = torch.empty_like(pi)
    nk = torch.empty((1,), dtype=torch.int32, device=r.device)
    check(lib().pcnn_nms_pose_fwd(ptr(r), ptr(pi), ptr(pp), ptr(nr), cap, cap, C, thresh, 1 if per_image else 0,
                                  ptr(keep), ptr(out_r), ptr(out_p), ptr(nk), stream()))
    return keep, out_r, out_p, nk


def nms(dets, thresh):
    """lib/utils/nms.py:3 — returns the kept row indices (int64 tensor, processing order).  Like the reference, the
    batch column is ignored."""
    d = require_cuda("dets", dets, torch.float32, 2)
    if d.shape[0] == 0:
        return torch.empty((0,), dtype=torch.int64, device=d.device)
    keep, _, _, nk = nms_pose_capacity(d, d, None, None, thresh, per_image=False)
    return keep[: int(nk.item())].to(torch.int64)
