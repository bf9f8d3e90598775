"""Host-side bindings of the pose-regression head kernels (include/posecnn_b200.h, csrc/fc_tc.cu):
RoiPool x2 + add (-> fp16 fc6 operand), and the fully connected layers as split-K wgmma GEMMs with fused
bias / ReLU / tanh (lib/networks/vgg16_convs.py:177-197, lib/networks/network.py:392-422)."""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, f32, lib, ptr, stream, workspace


def fc_weights_to_tc(w_in_out: torch.Tensor) -> torch.Tensor:
    """TF fc weights [in, out] f32 (network.py:404-406) -> [out padded to a multiple of 128][in] fp16 (K contiguous)."""
    k, n = w_in_out.shape
    npad = (n + 127) // 128 * 128
    w = torch.zeros((npad, k), dtype=torch.float16, device=w_in_out.device)
    w[:n] = w_in_out.t().to(torch.float16)
    return w.contiguous()


def roi_pool_pair(f5: torch.Tensor, f4: torch.Tensor, rois: torch.Tensor, pooled_h: int = 7, pooled_w: int = 7,
                  scale5: float = 1.0 / 16.0, scale4: float = 1.0 / 8.0, batch_offset: int = 0) -> torch.Tensor:
    """[N, pooled_h * pooled_w * C] fp16 = RoiPool(f5, scale5) + RoiPool(f4, scale4), flattened (h, w, c)."""
    assert f5.is_cuda and f5.dtype == torch.bfloat16 and f5.is_contiguous() and f4.dtype == torch.bfloat16 and f4.is_contiguous()
    assert rois.is_cuda and rois.dtype == torch.float32 and rois.is_contiguous() and rois.dim() == 2
    B, H5, W5, C = f5.shape
    _, H4, W4, C4 = f4.shape
    assert C4 == C and f4.shape[0] == B
    n = rois.shape[0]
    out = torch.empty((n, pooled_h * pooled_w * C), dtype=torch.float16, device=f5.device)
    check(lib().pcnn_roi_pool_pair_f16(ptr(f5), H5, W5, ptr(f4), H4, W4, C, B, int(batch_offset), ptr(rois), n, rois.shape[1],
                                        int(pooled_h), int(pooled_w), f32(scale5), f32(scale4), ptr(out), stream()))
    return out


def fc(a: torch.Tensor, w_tc: torch.Tensor, bias: torch.Tensor, act: str = "relu", out_dtype=torch.float16) -> torch.Tensor:
    """act(a @ w^T + bias).  a [M, K] fp16, w_tc = fc_weights_to_tc(W) [Npad, K] fp16, bias [n_valid] f32.
    out_dtype fp16 -> [M, Npad] (the next layer's operand; padding columns are zero), f32 -> [M, n_valid]."""
    assert a.is_cuda and a.dtype == torch.float16 and a.is_contiguous() and a.dim() == 2
    assert w_tc.dtype == torch.float16 and w_tc.is_contiguous() and bias.dtype == torch.float32
    M, K = a.shape
    N = w_tc.shape[0]
    assert w_tc.shape[1] == K
    nv = bias.numel()
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_fc_workspace_bytes(M, N, K, ctypes.byref(nbytes)))
    ws = workspace("fc", nbytes.value, a.device)
    code = {"none": 0, "relu": 1, "tanh": 2}[act]
    if out_dtype == torch.float16:
        out = torch.empty((M, N), dtype=torch.float16, device=a.device)
        check(lib().pcnn_fc_f16_tc(ptr(a), ptr(w_tc), ptr(bias), M, N, K, nv, code, ptr(out), N, ptr(None), ptr(ws),
                                    ctypes.c_size_t(ws.numel()), stream()))
    else:
        out = torch.empty((M, nv), dtype=torch.float32, device=a.device)
        check(lib().pcnn_fc_f16_tc(ptr(a), ptr(w_tc), ptr(bias), M, N, K, nv, code, ptr(None), 0, ptr(out), ptr(ws),
                                    ctypes.c_size_t(ws.numel()), stream()))
    return out
