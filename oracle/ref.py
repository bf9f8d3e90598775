"""ctypes front-end of oracle/_ref/libposecnn_ref.so — the reference's OWN CUDA kernels
(compiled unmodified from a checkout of the reference behind oracle/ref_shim; see oracle/ref_driver.cu).

TEST INFRASTRUCTURE ONLY (second oracle, SURVEY.md §8(c)).  Needs a GPU.  The library is
built by `make -C oracle ref` where a checkout of the reference exists; it is used to regenerate
tests/golden/ (tests/golden/make_golden.py), which the tests compare against.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libposecnn_ref.so")
_LIB = None
MAX_ROWS = 128 * 9


def available() -> bool:
    return os.path.exists(SO) and torch.cuda.is_available()


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(SO)
    return _LIB


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _f(x):
    return ctypes.c_float(float(x))


def _hough_common(fn_name, label, vertex, extents, meta, gt, is_train, vote_thr, per_thr, skip, want_votes):
    label = label.contiguous(); vertex = vertex.contiguous(); extents = extents.contiguous(); meta = meta.contiguous()
    B, H, W = label.shape
    C = vertex.shape[3] // 3
    dev = label.device
    if gt is None or gt.numel() == 0:
        gt_t, num_gt = torch.zeros((1, 13), device=dev), 0
    else:
        gt_t = gt.contiguous().reshape(-1, 13); num_gt = gt_t.shape[0]
    box = torch.zeros((MAX_ROWS, 7), device=dev); pose = torch.zeros((MAX_ROWS, 7), device=dev)
    target = torch.zeros((MAX_ROWS, 4 * C), device=dev); weight = torch.zeros((MAX_ROWS, 4 * C), device=dev)
    domain = torch.zeros((MAX_ROWS,), dtype=torch.int32, device=dev)
    nr_dev = torch.zeros((1,), dtype=torch.int32, device=dev)
    nr = ctypes.c_int(0)
    args = [_p(label), _p(vertex), _p(extents), _p(meta), _p(gt_t), B, H, W, C, num_gt, meta.shape[-1], int(is_train),
            _f(vote_thr), _f(per_thr), int(skip), _p(box), _p(pose), _p(target), _p(weight), _p(domain), _p(nr_dev),
            ctypes.byref(nr)]
    votes = None
    if fn_name == "ref_hough_canonical":
        votes = torch.zeros((B, C, H, W), device=dev) if want_votes else None
        args.append(_p(votes))
    torch.cuda.synchronize()
    rc = getattr(lib(), fn_name)(*args)
    assert rc == 0, fn_name
    n = max(1, nr.value)
    return (box[:n], pose[:n], target[:n], weight[:n], domain[:n]), nr.value, votes


def hough_full(label, vertex, extents, meta, gt, is_train, vote_thr, per_thr, skip):
    outs, n, _ = _hough_common("ref_hough_full", label, vertex, extents, meta, gt, is_train, vote_thr, per_thr, skip, False)
    return outs, n


def hough_canonical(label, vertex, extents, meta, gt, is_train, vote_thr, per_thr, skip, want_votes=True):
    return _hough_common("ref_hough_canonical", label, vertex, extents, meta, gt, is_train, vote_thr, per_thr, skip,
                         want_votes)


def roi_pool(data, rois, ph, pw, scale, pool_channel=0):
    data = data.contiguous(); rois = rois.contiguous()
    B, H, W, C = data.shape
    N, cr = rois.shape
    co = 1 if pool_channel else C
    top = torch.zeros((N, ph, pw, co), device=data.device)
    arg = torch.zeros((N, ph, pw, co), dtype=torch.int32, device=data.device)
    torch.cuda.synchronize()
    assert lib().ref_roi_pool_fwd(_p(data), _p(rois), N, cr, H, W, C, ph, pw, _f(scale), int(pool_channel), _p(top),
                                  _p(arg)) == 0
    return top, arg


def roi_pool_grad(data, rois, argmax, grad, ph, pw, scale, pool_channel=0):
    B, H, W, C = data.shape
    N, cr = rois.shape
    out = torch.zeros_like(data)
    torch.cuda.synchronize()
    assert lib().ref_roi_pool_bwd(_p(grad.contiguous()), _p(argmax.contiguous()), _p(rois.contiguous()), B, N, cr, H, W, C,
                                  ph, pw, _f(scale), int(pool_channel), _p(out)) == 0
    return out


def hard_label(prob, gt, threshold):
    prob = prob.contiguous(); gt = gt.contiguous()
    B, H, W, C = prob.shape
    top = torch.zeros_like(prob)
    torch.cuda.synchronize()
    assert lib().ref_hard_label_fwd(_p(prob), _p(gt), B, H, W, C, _f(threshold), _p(top)) == 0
    return top


def backproject(data, label, depth, meta, label_3d, G, ks, thr):
    B, H, W, Cf = data.shape
    C = label.shape[3]
    dev = data.device
    td = torch.zeros((B, G, G, G, Cf), device=dev); tl = torch.zeros((B, G, G, G, C), device=dev)
    tf = torch.zeros((B, G, G, G, Cf), device=dev)
    torch.cuda.synchronize()
    assert lib().ref_backproject_fwd(_p(data.contiguous()), _p(label.contiguous()), _p(depth.contiguous()),
                                     _p(meta.contiguous()), _p(label_3d.contiguous()), B, H, W, Cf, C, meta.shape[-1], G,
                                     ks, _f(thr), _p(td), _p(tl), _p(tf)) == 0
    return td, tl, tf


def backproject_grad(top_diff, depth, meta, H, W):
    B, G = top_diff.shape[0], top_diff.shape[1]
    Cf = top_diff.shape[4]
    out = torch.zeros((B, H, W, Cf), device=top_diff.device)
    torch.cuda.synchronize()
    assert lib().ref_backproject_bwd(_p(top_diff.contiguous()), _p(depth.contiguous()), _p(meta.contiguous()), B, H, W, Cf,
                                     meta.shape[-1], G, _p(out)) == 0
    return out


def project(data, depth, meta):
    B, G = data.shape[0], data.shape[1]
    Cf = data.shape[4]
    H, W = depth.shape[1], depth.shape[2]
    out = torch.zeros((B, H, W, Cf), device=data.device)
    torch.cuda.synchronize()
    assert lib().ref_project_fwd(_p(data.contiguous()), _p(depth.contiguous()), _p(meta.contiguous()), B, H, W, Cf,
                                 meta.shape[-1], G, _p(out)) == 0
    return out


def project_grad(top_diff, depth, meta, G, ks, thr):
    B, H, W, Cf = top_diff.shape
    out = torch.zeros((B, G, G, G, Cf), device=top_diff.device)
    torch.cuda.synchronize()
    assert lib().ref_project_bwd(_p(top_diff.contiguous()), _p(depth.contiguous()), _p(meta.contiguous()), B, H, W, Cf,
                                 meta.shape[-1], G, ks, _f(thr), _p(out)) == 0
    return out


def average_distance_loss(pred, target, weight, point, symmetry, margin):
    N = pred.shape[0]
    C, P = point.shape[0], point.shape[1]
    loss = torch.zeros((1,), device=pred.device)
    diff = torch.zeros_like(pred)
    torch.cuda.synchronize()
    assert lib().ref_average_distance_fwd(_p(pred.contiguous()), _p(target.contiguous()), _p(weight.contiguous()),
                                          _p(point.contiguous()), _p(symmetry.contiguous()), N, C, P, _f(margin),
                                          _p(loss), _p(diff)) == 0
    return loss, diff
