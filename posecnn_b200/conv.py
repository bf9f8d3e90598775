"""Host-side bindings of the tensor-core convolution stack (include/posecnn_b200.h,
posecnn_b200/csrc/conv_tc.cu).  Activations are NHWC torch.bfloat16 CUDA tensors."""
from __future__ import annotations

import torch

from ._lib import check, lib, ptr, stream


def hwio_to_tc(weights_hwio: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """TF filter layout [kh, kw, Cin, Cout] f32 (network.py:166-170) -> [Cout][kh*kw*Cin] bf16 (or `dtype`)."""
    kh, kw, ci, co = weights_hwio.shape
    return weights_hwio.permute(3, 0, 1, 2).reshape(co, kh * kw * ci).to(dtype).contiguous()


def hwio_to_tc_dgrad(weights_hwio: torch.Tensor) -> torch.Tensor:
    """Weights for the INPUT-gradient pass of a SAME / stride-1 convolution, in the layout `conv_bf16` consumes:
    d x = conv(d y, W') with W'[r, s, co, ci] = W[k-1-r, k-1-s, ci, co] (taps flipped, channels transposed), so the
    backward-data pass of every trunk layer is the forward tensor-core kernel on these weights (zero bias, no ReLU;
    the ReLU mask of the layer below multiplies the result).  Returns [Cin][k*k*Cout] bf16."""
    kh, kw, ci, co = weights_hwio.shape
    flipped = torch.flip(weights_hwio, dims=(0, 1)).permute(0, 1, 3, 2).contiguous()      # [kh, kw, co, ci] = HWIO of the dgrad conv
    return hwio_to_tc(flipped)


def conv_bf16(x: torch.Tensor, w_tc: torch.Tensor, bias: torch.Tensor, ksize: int, relu: bool, block_n: int = 0,
              out: torch.Tensor | None = None) -> torch.Tensor:
    """x [B,H,W,Cin] bf16, w_tc [Cout, k*k*Cin] bf16, bias [Cout] f32 -> [B,H,W,Cout] bf16."""
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4
    assert w_tc.dtype == torch.bfloat16 and w_tc.is_contiguous() and bias.dtype == torch.float32
    B, H, W, Cin = x.shape
    Cout = w_tc.shape[0]
    assert w_tc.shape[1] == ksize * ksize * Cin
    if out is None:
        out = torch.empty((B, H, W, Cout), dtype=torch.bfloat16, device=x.device)
    check(lib().pcnn_conv_bf16_tc(ptr(x), ptr(w_tc), ptr(bias), ptr(out), B, H, W, Cin, Cout, int(ksize), int(bool(relu)),
                                  int(block_n), stream()))
    return out


def conv_pool_bf16(x: torch.Tensor, w_tc: torch.Tensor, bias: torch.Tensor, ksize: int, relu: bool, block_n: int = 0) -> torch.Tensor:
    """conv + bias + ReLU + 2x2/2 max pool in one kernel: x [B,H,W,Cin] bf16 -> [B,H/2,W/2,Cout] bf16."""
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4
    B, H, W, Cin = x.shape
    Cout = w_tc.shape[0]
    out = torch.empty((B, H // 2, W // 2, Cout), dtype=torch.bfloat16, device=x.device)
    check(lib().pcnn_conv_pool_bf16_tc(ptr(x), ptr(w_tc), ptr(bias), ptr(out), B, H, W, Cin, Cout, int(ksize), int(bool(relu)),
                                       int(block_n), stream()))
    return out


def conv3x3_small_cin(x: torch.Tensor, w_hwio: torch.Tensor, bias: torch.Tensor, relu: bool = True) -> torch.Tensor:
    """conv1_1: x [B,H,W,3] f32, w [3,3,3,Cout] f32 -> [B,H,W,Cout] bf16."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
    B, H, W, Cin = x.shape
    Cout = w_hwio.shape[3]
    out = torch.empty((B, H, W, Cout), dtype=torch.bfloat16, device=x.device)
    check(lib().pcnn_conv3x3_small_cin(ptr(x), ptr(w_hwio.contiguous()), ptr(bias), ptr(out), B, H, W, Cin, Cout,
                                       int(bool(relu)), stream()))
    return out


def maxpool2x2(x: torch.Tensor) -> torch.Tensor:
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous()
    B, H, W, C = x.shape
    out = torch.empty((B, H // 2, W // 2, C), dtype=torch.bfloat16, device=x.device)
    check(lib().pcnn_maxpool2x2_bf16(ptr(x), ptr(out), B, H, W, C, stream()))
    return out


def im2col_c3(x: torch.Tensor, mean=None) -> torch.Tensor:
    """First layer: x [B,H,W,3] f32 or u8 -> [B,H,W,64] bf16 (K = tap*3 + c, zero padded to 64)."""
    import ctypes
    assert x.is_cuda and x.is_contiguous() and x.shape[3] == 3 and x.dtype in (torch.float32, torch.uint8)
    B, H, W, _ = x.shape
    out = torch.empty((B, H, W, 64), dtype=torch.bfloat16, device=x.device)
    m = (ctypes.c_float * 3)(*(mean if mean is not None else (0.0, 0.0, 0.0)))
    check(lib().pcnn_im2col_c3(ptr(x), int(x.dtype == torch.uint8), m, ptr(out), B, H, W, stream()))
    return out


def im2col_depth(depth: torch.Tensor, mean) -> torch.Tensor:
    """First layer of the depth trunk: depth [B,H,W] f32 (raw, sensor units) -> [B,H,W,64] bf16, the im2col view (K = tap*3 + c)
    of the blob clip(d / 2000, 0, 1) * 255 tiled x3 - mean, formed as conv1_depth_fused forms it (the conv1_1_p weight-gradient input)."""
    import ctypes
    assert depth.is_cuda and depth.is_contiguous() and depth.dtype == torch.float32 and depth.dim() == 3
    B, H, W = depth.shape
    out = torch.empty((B, H, W, 64), dtype=torch.bfloat16, device=depth.device)
    m = (ctypes.c_float * 3)(*mean)
    check(lib().pcnn_im2col_depth(ptr(depth), m, ptr(out), B, H, W, stream()))
    return out


def conv1_1_weights_to_tc(w_hwio: torch.Tensor) -> torch.Tensor:
    """[3,3,3,Cout] f32 -> [Cout, 64] bf16 matching im2col_c3's K order (tap*3 + c)."""
    co = w_hwio.shape[3]
    w = torch.zeros((co, 64), dtype=torch.float32, device=w_hwio.device)
    w[:, :27] = w_hwio.reshape(27, co).t()
    return w.to(torch.bfloat16).contiguous()


def conv1_fused(x: torch.Tensor, w_tc64: torch.Tensor, bias: torch.Tensor, mean=None, relu: bool = True) -> torch.Tensor:
    """conv1_1 in one kernel: x [B,H,W,3] u8 / f32, w_tc64 = conv1_1_weights_to_tc(w) [64,64] bf16 -> [B,H,W,64] bf16."""
    import ctypes
    assert x.is_cuda and x.is_contiguous() and x.shape[3] == 3 and x.dtype in (torch.float32, torch.uint8)
    assert w_tc64.shape == (64, 64) and w_tc64.dtype == torch.bfloat16
    B, H, W, _ = x.shape
    out = torch.empty((B, H, W, 64), dtype=torch.bfloat16, device=x.device)
    m = (ctypes.c_float * 3)(*(mean if mean is not None else (0.0, 0.0, 0.0)))
    check(lib().pcnn_conv1_fused_tc(ptr(x), int(x.dtype == torch.uint8), m, ptr(w_tc64), ptr(bias), ptr(out), B, H, W,
                                    int(bool(relu)), stream()))
    return out


def conv1_depth_fused(depth: torch.Tensor, w_tc64: torch.Tensor, bias: torch.Tensor, mean, relu: bool = True) -> torch.Tensor:
    """conv1_1_p on a raw depth image: depth [B,H,W] f32 (sensor units) -> [B,H,W,64] bf16; the depth blob of
    lib/fcn/test.py:70-76 (clip(d / 2000, 0, 1) * 255 tiled x3 - PIXEL_MEANS) is formed inside the kernel's loader."""
    import ctypes
    assert depth.is_cuda and depth.is_contiguous() and depth.dtype == torch.float32 and depth.dim() == 3
    B, H, W = depth.shape
    out = torch.empty((B, H, W, 64), dtype=torch.bfloat16, device=depth.device)
    m = (ctypes.c_float * 3)(*mean)
    check(lib().pcnn_conv1_depth_fused_tc(ptr(depth), m, ptr(w_tc64), ptr(bias), ptr(out), B, H, W, int(bool(relu)), stream()))
    return out
