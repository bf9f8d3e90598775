"""Averagedistance / AveragedistanceGrad — drop-in for lib/average_distance_loss/average_distance_loss_op.py.

Registration: average_distance_loss_op.cc:38-54.  Call site lib/networks/network.py:238:
average_distance_loss(prediction [N,4C], target [N,4C], weight [N,4C], point [C,P,3],
symmetry [C], margin) -> (loss [1], bottom_diff [N,4C]).
"""
from __future__ import annotations

import ctypes

import torch

try:
    from .._lib import check, lib, ptr, require_cuda, stream, workspace
except ImportError:
    from posecnn_b200._lib import check, lib, ptr, require_cuda, stream, workspace


def average_distance_loss(bottom_prediction, bottom_target, bottom_weight, bottom_point, bottom_symmetry, margin,
                          name=None):
    pred = require_cuda("bottom_prediction", bottom_prediction, torch.float32, 2)  # average_distance_loss_op.cc:264-265
    target = require_cuda("bottom_target", bottom_target, torch.float32, 2)        # :269-270
    weight = require_cuda("bottom_weight", bottom_weight, torch.float32, 2)        # :274-275
    point = require_cuda("bottom_point", bottom_point, torch.float32, 3)           # :279-280
    symmetry = require_cuda("bottom_symmetry", bottom_symmetry, torch.float32, 1)  # :284-285
    N, ch = pred.shape
    C, P = point.shape[0], point.shape[1]
    if ch != 4 * C or target.shape != pred.shape or weight.shape != pred.shape:
        raise ValueError("prediction/target/weight must be [N, 4*num_classes]")
    loss = torch.empty((1,), dtype=torch.float32, device=pred.device)
    diff = torch.empty_like(pred)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_average_distance_workspace_bytes(N, ctypes.byref(nbytes)))
    ws = workspace("avgdist", nbytes.value, pred.device)
    check(lib().pcnn_average_distance_fwd(ptr(pred), ptr(target), ptr(weight), ptr(point), ptr(symmetry), N, C, P, margin, ptr(loss),
                                          ptr(diff), ptr(ws), ws.numel(), stream()))
    return loss, diff


averagedistance = average_distance_loss


def average_distance_loss_grad(bottom_diff, grad, margin=None, name=None):
    diff = require_cuda("bottom_diff", bottom_diff, torch.float32, 2)
    grad = require_cuda("grad", grad, torch.float32)
    out = torch.empty_like(diff)
    check(lib().pcnn_average_distance_bwd(ptr(grad), ptr(diff), diff.shape[0], diff.shape[1], ptr(out), stream()))
    return out


averagedistance_grad = average_distance_loss_grad
