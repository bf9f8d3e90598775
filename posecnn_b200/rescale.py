"""Image scale on the device: the SCALES_BASE resizes of the reference (csrc/rescale.cu).

The LINEMOD object-coordinate models (experiments/cfgs/linemod_<object>_3d.yml) set TRAIN.SCALES_BASE and TEST.SCALES_BASE to
(1.5,): the reference resizes every 480 x 640 frame to 720 x 960 with cv2.resize before the network and resizes the predicted
labels back afterwards.  These functions do the same resizes on the device, with OpenCV's generic arithmetic bit for bit, and
hold the per-tensor policy (which tensor, which interpolation, which rounding) in one place:

  colour frame (test)   color_blob      f32(u8) - PIXEL_MEANS, LINEAR                      lib/fcn/test.py:49-65
  raw depth (test)      resize_depth    LINEAR, rounded and saturated to uint16 units      test.py:1335, 1384
  labels back (test)    resize_nearest  NEAREST at 1 / s                                   test.py:1421
  training inputs       training_inputs colour blob LINEAR, label NEAREST, vertmap LINEAR,  gt_synthesize_layer/minibatch.py:179-183,
                                        centres (cx, cy) * s                               352, 416, 435

vgg16_convs.forward, GraphedForward and Trainer take their inputs at the network's resolution; intrinsics scale through
train_ops.pack_pose_meta(..., im_scale=s) and record boxes through the network's `scales`.  Every function takes the float64 factor
s the configuration gives and produces round(H s) x round(W s) (half to even).
"""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, lib, ptr, require_cuda, stream
from .networks.vgg16_convs import PIXEL_MEANS


def scaled_size(H: int, W: int, s: float) -> tuple:
    """(round(H s), round(W s)) with round half to even: cv2.resize's destination size for fx = fy = s."""
    s = float(s)
    if not (s > 0.0 and s < float("inf")):
        raise ValueError(f"scale must be finite and > 0 (got {s})")
    return round(H * s), round(W * s)


def _out(x: torch.Tensor, s: float):
    B, H, W = x.shape[:3]
    Ho, Wo = scaled_size(H, W, s)
    return B, H, W, Ho, Wo


def color_blob(frames_u8: torch.Tensor, s: float, mean=PIXEL_MEANS) -> torch.Tensor:
    """frames [B,H,W,3] u8 BGR -> the test-time colour blob [B,Ho,Wo,3] f32: f32(u8) - mean (float64 means, as numpy), resized
    LINEAR (pcnn_resize_color_u8)."""
    frames_u8 = require_cuda("frames", frames_u8, torch.uint8, 4)
    if frames_u8.shape[3] != 3:
        raise ValueError("frames must be [B,H,W,3]")
    B, H, W, Ho, Wo = _out(frames_u8, s)
    out = torch.empty((B, Ho, Wo, 3), dtype=torch.float32, device=frames_u8.device)
    m = (ctypes.c_double * 3)(*[float(v) for v in mean])
    check(lib().pcnn_resize_color_u8(ptr(frames_u8), B, H, W, float(s), Ho, Wo, m, ptr(out), stream()))
    return out


def resize_linear(x: torch.Tensor, s: float) -> torch.Tensor:
    """x [B,H,W] or [B,H,W,C] f32 (C = 1 or 3: a colour blob, a vertmap) -> the same rank at round(H s) x round(W s), LINEAR
    (pcnn_resize_linear_f32)."""
    x = require_cuda("x", x, torch.float32, (3, 4))
    C = x.shape[3] if x.dim() == 4 else 1
    if C not in (1, 3):
        raise ValueError("x must have 1 or 3 channels")
    B, H, W, Ho, Wo = _out(x, s)
    out = torch.empty((B, Ho, Wo) + tuple(x.shape[3:]), dtype=torch.float32, device=x.device)
    check(lib().pcnn_resize_linear_f32(ptr(x), B, H, W, C, float(s), Ho, Wo, ptr(out), stream()))
    return out


def resize_depth(depth: torch.Tensor, s: float) -> torch.Tensor:
    """Raw depth [B,H,W] torch.uint16, or f32 holding integer sensor units -> the same dtype at round(H s) x round(W s): LINEAR,
    rounded half to even and saturated to [0, 65535] as cv2 does on the uint16 image (pcnn_resize_depth)."""
    if not isinstance(depth, torch.Tensor) or depth.dtype not in (torch.uint16, torch.float32):
        raise TypeError("depth must be a torch.uint16 or torch.float32 tensor")
    depth = require_cuda("depth", depth, depth.dtype, 3)
    B, H, W, Ho, Wo = _out(depth, s)
    out = torch.empty((B, Ho, Wo), dtype=depth.dtype, device=depth.device)
    check(lib().pcnn_resize_depth(ptr(depth), int(depth.dtype == torch.uint16), B, H, W, float(s), Ho, Wo, ptr(out), stream()))
    return out


def resize_nearest(label: torch.Tensor, s: float) -> torch.Tensor:
    """Label map [B,H,W] int32 -> [B,round(H s),round(W s)] int32, NEAREST (pcnn_resize_nearest_i32).  The predicted labels go back
    to the frame with s = 1 / SCALES_BASE[0], as test.py:1421 passes it."""
    label = require_cuda("label", label, torch.int32, 3)
    B, H, W, Ho, Wo = _out(label, s)
    out = torch.empty((B, Ho, Wo), dtype=torch.int32, device=label.device)
    check(lib().pcnn_resize_nearest_i32(ptr(label), B, H, W, float(s), Ho, Wo, ptr(out), stream()))
    return out


def training_inputs(blob: torch.Tensor, gt_label_2d: torch.Tensor, centers: torch.Tensor, s: float,
                    vertmap: torch.Tensor | None = None) -> dict:
    """The data layer's scaled tensors (minibatch.py:179-183, 352, 416, 435) from their frame-resolution forms: blob [B,H,W,3] f32
    (augment.augment_color's output: composited, jittered, noised, minus PIXEL_MEANS) LINEAR; gt_label_2d [B,H,W] int32 NEAREST
    (before or after the two-class remap: it is per pixel); centers [B,C,3] = (cx, cy, z) with cx, cy times s in float32 (z is a
    depth, not a pixel coordinate); vertmap [B,H,W,3] f32 LINEAR.  Returns {data, gt_label_2d, centers, vertmap} for Trainer.step;
    form the meta with train_ops.pack_pose_meta(..., im_scale=s)."""
    centers = require_cuda("centers", centers, torch.float32, 3)
    if centers.shape[2] != 3 or centers.shape[0] != blob.shape[0]:
        raise ValueError("centers must be [B,C,3]")
    if blob.dim() != 4 or tuple(gt_label_2d.shape) != tuple(blob.shape[:3]) or \
            (vertmap is not None and tuple(vertmap.shape) != tuple(blob.shape[:3]) + (3,)):
        raise ValueError("blob [B,H,W,3], gt_label_2d [B,H,W] and vertmap [B,H,W,3] must share B, H, W")
    scaled = torch.cat([centers[..., :2] * float(s), centers[..., 2:]], 2)              # float32 products, as numpy's im_scale * center
    return {"data": resize_linear(blob, s), "gt_label_2d": resize_nearest(gt_label_2d, s), "centers": scaled,
            "vertmap": None if vertmap is None else resize_linear(vertmap, s)}
