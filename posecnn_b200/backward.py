"""Host-side bindings of the backward-pass kernels (include/posecnn_b200.h, csrc/wgrad_tc.cu): weight gradients on the
tensor cores, ReLU-mask / max-pool routing with bias gradients, gradient fan-in.  Activations NHWC torch.bfloat16."""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, lib, ptr, stream, workspace


def conv_wgrad(x: torch.Tensor, dz: torch.Tensor, ksize: int, scale: float = 1.0, w_master: torch.Tensor | None = None,
               decay: float = 0.0, out: torch.Tensor | None = None) -> torch.Tensor:
    """dW [Cout, k*k*Cin] f32 (tensor-core weight layout) = scale * sum_pixels x (*) dz (+ decay * w_master).
    x [B,H,W,Cin], dz [B,H,W,Cout] bf16; a fully connected layer passes [1,1,rows,C] views."""
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4
    assert dz.dtype == torch.bfloat16 and dz.is_contiguous() and dz.shape[:3] == x.shape[:3]
    B, H, W, Cin = x.shape
    Cout = dz.shape[3]
    if out is None:
        out = torch.empty((Cout, ksize * ksize * Cin), dtype=torch.float32, device=x.device)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_conv_wgrad_workspace_bytes(B, H, W, Cin, Cout, int(ksize), ctypes.byref(nbytes)))
    ws = workspace("wgrad", nbytes.value, x.device)
    check(lib().pcnn_conv_wgrad_bf16_tc(ptr(x), ptr(dz), B, H, W, Cin, Cout, int(ksize), scale, ptr(w_master), decay, ptr(out),
                                        ptr(ws), ws.numel(), stream()))
    return out


def _bias_ws(C, device):
    n = ctypes.c_size_t(0)
    check(lib().pcnn_bias_ws_bytes(int(C), ctypes.byref(n)))
    return workspace("bias_grad", n.value, device)


def relu_bwd(g: torch.Tensor, y: torch.Tensor | None, has_relu: bool = True, want_bias: bool = False, scale: float = 1.0,
             bias: torch.Tensor | None = None, decay: float = 0.0, want_dz: bool = True):
    """dz = g * [y > 0] (or g when the layer has no ReLU); optional bias gradient [C] f32 = scale * sum_pixels dz (+ decay * bias)."""
    assert g.is_cuda and g.dtype == torch.bfloat16 and g.is_contiguous()
    C = g.shape[-1]
    npix = g.numel() // C
    dz = torch.empty_like(g) if want_dz else None
    db = torch.empty((C,), dtype=torch.float32, device=g.device) if want_bias else None
    ws = _bias_ws(C, g.device) if want_bias else None
    check(lib().pcnn_relu_bwd_bf16(ptr(g), ptr(y), npix, C, int(bool(has_relu)), ptr(dz), scale, ptr(bias), decay,
                                   ptr(db), ptr(ws), ws.numel() if ws is not None else 0, stream()))
    return (dz, db) if want_bias else dz


def maxpool_relu_bwd(g: torch.Tensor, y: torch.Tensor, want_bias: bool = False, scale: float = 1.0, bias: torch.Tensor | None = None,
                     decay: float = 0.0):
    """g [B,H/2,W/2,C] (gradient of the pooled tensor), y [B,H,W,C] (pre-pool, post-ReLU) -> dz [B,H,W,C]: the gradient routed
    to each window's first maximum and masked by the ReLU of the convolution below the pool."""
    assert g.is_cuda and g.dtype == torch.bfloat16 and g.is_contiguous() and y.dtype == torch.bfloat16 and y.is_contiguous()
    B, H, W, C = y.shape
    dz = torch.empty_like(y)
    db = torch.empty((C,), dtype=torch.float32, device=g.device) if want_bias else None
    ws = _bias_ws(C, g.device) if want_bias else None
    check(lib().pcnn_maxpool_relu_bwd_bf16(ptr(g), ptr(y), B, H, W, C, ptr(dz), scale, ptr(bias), decay, ptr(db), ptr(ws),
                                           ws.numel() if ws is not None else 0, stream()))
    return (dz, db) if want_bias else dz


def add_to_bf16(a: torch.Tensor, b: torch.Tensor | None = None, b_f32: torch.Tensor | None = None) -> torch.Tensor:
    """a + b (+ b_f32) -> bf16 (gradient fan-in of conv4_3 / conv5_3)."""
    assert a.is_cuda and a.dtype == torch.bfloat16 and a.is_contiguous() and a.numel() % 8 == 0
    out = torch.empty_like(a)
    check(lib().pcnn_add_to_bf16(ptr(a), ptr(b), ptr(b_f32), a.numel(), ptr(out), stream()))
    return out
