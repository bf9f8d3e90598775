"""Project / ProjectGrad — drop-in for lib/projecting_layer/projecting_op.py.

Registration: projecting_op.cc:30-47.  Call site lib/networks/network.py:246:
project(data [B,G,G,G,Cf], depth [B,H,W,1], meta [B,1,1,48], kernel_size, threshold) -> [B,H,W,Cf].
"""
from __future__ import annotations

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream
except ImportError:
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream


def project(bottom_data, bottom_depth, bottom_meta_data, kernel_size, threshold, name=None):
    data = require_cuda("bottom_data", bottom_data, torch.float32, 5)         # projecting_op.cc:240-241
    depth = require_cuda("bottom_depth", bottom_depth, torch.float32, (3, 4)) # :245-246
    meta = require_cuda("bottom_meta_data", bottom_meta_data, torch.float32)  # :249-250
    B, G = data.shape[0], data.shape[1]
    Cf = data.shape[4]
    H, W = depth.shape[1], depth.shape[2]
    top = torch.empty((B, H, W, Cf), dtype=torch.float32, device=data.device)
    check(lib().pcnn_project_fwd(ptr(data), ptr(depth), ptr(meta), B, H, W, Cf, meta.shape[-1], G, ptr(top), stream()))
    return top


def project_grad(bottom_data, bottom_depth, bottom_meta_data, grad, kernel_size, threshold, name=None):
    data = require_cuda("bottom_data", bottom_data, torch.float32, 5)
    depth = require_cuda("bottom_depth", bottom_depth, torch.float32, (3, 4))
    meta = require_cuda("bottom_meta_data", bottom_meta_data, torch.float32)
    grad = require_cuda("grad", grad, torch.float32, 4)
    B, G = data.shape[0], data.shape[1]
    Cf = data.shape[4]
    H, W = depth.shape[1], depth.shape[2]
    out = torch.empty_like(data)
    check(lib().pcnn_project_bwd(ptr(grad), ptr(depth), ptr(meta), B, H, W, Cf, meta.shape[-1], G, int(kernel_size),
                                 threshold, ptr(out), stream()))
    return out
