"""RoiPool / RoiPoolGrad — drop-in for lib/roi_pooling_layer/roi_pooling_op.py.

Registration: roi_pooling_op.cc:29-50.  Call site lib/networks/network.py:327-332:
roi_pool(data [B,H,W,C], rois [N,>=6] rows [b, cls, x1,y1,x2,y2,...], pooled_height,
pooled_width, spatial_scale, pool_channel) -> (top [N,ph,pw,C], argmax [N,ph,pw,C] int32).
"""
from __future__ import annotations

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream
except ImportError:
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream


def roi_pool(bottom_data, bottom_rois, pooled_height, pooled_width, spatial_scale, pool_channel=0, name=None):
    if isinstance(bottom_data, torch.Tensor) and bottom_data.dtype == torch.bfloat16 and not pool_channel:
        # activation format of the tensor-core trunk; same semantics, fp32 outputs
        data = require_cuda("bottom_data", bottom_data, torch.bfloat16, 4)
        rois = require_cuda("bottom_rois", bottom_rois, torch.float32, 2)
        B, H, W, C = data.shape
        N, cr = rois.shape
        top = torch.empty((N, pooled_height, pooled_width, C), dtype=torch.float32, device=data.device)
        argmax = torch.empty((N, pooled_height, pooled_width, C), dtype=torch.int32, device=data.device)
        check(lib().pcnn_roi_pool_fwd_bf16(ptr(data), ptr(rois), N, cr, B, H, W, C, int(pooled_height), int(pooled_width),
                                           spatial_scale, ptr(top), ptr(argmax), stream()))
        return top, argmax
    data = require_cuda("bottom_data", bottom_data, torch.float32, 4)   # roi_pooling_op.cc:297-298
    rois = require_cuda("bottom_rois", bottom_rois, torch.float32, 2)   # roi_pooling_op.cc:301-302
    B, H, W, C = data.shape
    N, cr = rois.shape
    co = 1 if pool_channel else C
    top = torch.empty((N, pooled_height, pooled_width, co), dtype=torch.float32, device=data.device)
    argmax = torch.empty((N, pooled_height, pooled_width, co), dtype=torch.int32, device=data.device)
    check(lib().pcnn_roi_pool_fwd(ptr(data), ptr(rois), N, cr, B, H, W, C, int(pooled_height), int(pooled_width),
                                  spatial_scale, int(pool_channel), ptr(top), ptr(argmax), stream()))
    return top, argmax


def roi_pool_grad(bottom_data, bottom_rois, argmax, grad, pooled_height, pooled_width, spatial_scale, pool_channel=0,
                  name=None):
    # bottom_data only supplies the shape (RoiPoolGrad reads no feature values, roi_pooling_op_gpu.cu.cc:134-229): it
    # may be the trunk's bf16 activation; the gradient is float32 like the reference's
    if not (isinstance(bottom_data, torch.Tensor) and bottom_data.is_cuda and bottom_data.dim() == 4):
        raise RuntimeError("bottom_data must be a 4-dimensional CUDA tensor (posecnn_b200 has no CPU path)")
    rois = require_cuda("bottom_rois", bottom_rois, torch.float32, 2)
    argmax = require_cuda("argmax", argmax, torch.int32, 4)
    grad = require_cuda("grad", grad, torch.float32, 4)
    B, H, W, C = bottom_data.shape
    N, cr = rois.shape
    out = torch.empty((B, H, W, C), dtype=torch.float32, device=bottom_data.device)
    check(lib().pcnn_roi_pool_bwd(ptr(grad), ptr(argmax), ptr(rois), B, N, cr, H, W, C, int(pooled_height),
                                  int(pooled_width), spatial_scale, int(pool_channel), ptr(out), stream()))
    return out
