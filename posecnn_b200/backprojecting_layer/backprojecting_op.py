"""Backproject / BackprojectGrad — drop-in for lib/backprojecting_layer/backprojecting_op.py.

Registration: backprojecting_op.cc:30-53.  Call site lib/networks/network.py:226:
backproject(data [B,H,W,Cf], label [B,H,W,C], depth [B,H,W,1], meta [B,1,1,48],
label_3d [B,G,G,G,C], grid_size, kernel_size, threshold)
 -> (top_data [B,G,G,G,Cf], top_label [B,G,G,G,C], top_flag [B,G,G,G,Cf]).
"""
from __future__ import annotations

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream
except ImportError:
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream


def backproject(bottom_data, bottom_label, bottom_depth, bottom_meta_data, bottom_label_3d, grid_size, kernel_size,
                threshold, name=None):
    data = require_cuda("bottom_data", bottom_data, torch.float32, 4)         # backprojecting_op.cc:333-334
    label = require_cuda("bottom_label", bottom_label, torch.float32, 4)      # :338-339
    depth = require_cuda("bottom_depth", bottom_depth, torch.float32, (3, 4)) # :342-343
    meta = require_cuda("bottom_meta_data", bottom_meta_data, torch.float32)  # :346-347
    label_3d = require_cuda("bottom_label_3d", bottom_label_3d, torch.float32, 5)  # :350-351
    B, H, W, Cf = data.shape
    C = label.shape[3]
    G = int(grid_size)
    dev = data.device
    top_data = torch.empty((B, G, G, G, Cf), dtype=torch.float32, device=dev)
    top_label = torch.empty((B, G, G, G, C), dtype=torch.float32, device=dev)
    top_flag = torch.empty((B, G, G, G, Cf), dtype=torch.float32, device=dev)
    check(lib().pcnn_backproject_fwd(ptr(data), ptr(label), ptr(depth), ptr(meta), ptr(label_3d), B, H, W, Cf, C, meta.shape[-1], G,
                                     int(kernel_size), threshold, ptr(top_data), ptr(top_label), ptr(top_flag), stream()))
    return top_data, top_label, top_flag


def backproject_grad(bottom_data, bottom_depth, bottom_meta_data, grad, grid_size, kernel_size=None, threshold=None,
                     name=None):
    data = require_cuda("bottom_data", bottom_data, torch.float32, 4)
    depth = require_cuda("bottom_depth", bottom_depth, torch.float32, (3, 4))
    meta = require_cuda("bottom_meta_data", bottom_meta_data, torch.float32)
    grad = require_cuda("grad", grad, torch.float32, 5)
    B, H, W, Cf = data.shape
    out = torch.empty_like(data)
    check(lib().pcnn_backproject_bwd(ptr(grad), ptr(depth), ptr(meta), B, H, W, Cf, meta.shape[-1], int(grid_size), ptr(out), stream()))
    return out
