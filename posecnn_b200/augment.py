"""Training image blobs on the device: the image side of the synthetic-data loader (lib/gt_synthesize_layer/minibatch.py:147-200).

For lov_color_2d.yml (SYNTHESIZE, CHROMATIC, ADD_NOISE) the reference builds each image's blob on the host: it pastes a random
background where the rendered alpha is 0, runs chromatic_transform (lib/utils/blob.py:74-99) and add_noise (blob.py:102-129), and
subtracts PIXEL_MEANS.  augment_color does all four in one launch (csrc/augment.cu); depth_blob_train forms the RGB-D network's
training depth blob d / max(d) * 255 with its own noise.  Both return the float32 blob Trainer.forward accepts (data= / data_p=).

The per-image random scalars come from draw_params, with the reference's formulas and its numpy RandomState call order; the Gaussian
field comes from a counter-based generator keyed per image (or from a caller-supplied field, bit for bit).
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from ._lib import check, lib, ptr, require_cuda, stream
from .networks.vgg16_convs import PIXEL_MEANS

# columns of the parameter table (PCNN_AUG_* in include/posecnn_b200.h)
COLUMNS = ("background", "chromatic", "d_h", "d_l", "d_s", "noise", "sigma", "blur_size", "blur_axis")
NUM_PARAMS = len(COLUMNS)
NOISE_NONE, NOISE_GAUSS, NOISE_BLUR = 0, 1, 2
BLUR_SIZES = (3, 5, 7, 9, 11, 15)                               # add_noise's `sizes` (blob.py:120)


def _draw_noise(rng, row):
    """add_noise's draws (blob.py:105-127) without the H x W field: r; then var (Gaussian) or the size index and orientation (blur)."""
    if rng.rand(1)[0] < 0.9:
        var = rng.rand(1) * 0.3 * 256
        row[5], row[6] = NOISE_GAUSS, float((var ** 0.5)[0])
    else:
        row[5], row[7] = NOISE_BLUR, BLUR_SIZES[int(rng.randint(len(BLUR_SIZES), size=1)[0])]
        row[8] = 0.0 if rng.rand(1)[0] < 0.5 else 1.0           # middle kernel ROW of ones = along the row


def validate_params(table: np.ndarray, n_backgrounds: int) -> None:
    """Host check of a parameter table [B, NUM_PARAMS] (the kernel never faults on a bad row, but it silently treats one as 'none')."""
    t = np.asarray(table, dtype=np.float64)
    if t.ndim != 2 or t.shape[1] != NUM_PARAMS:
        raise ValueError(f"parameter table must be [B, {NUM_PARAMS}], got {t.shape}")
    if not np.isfinite(t).all():
        raise ValueError("parameter table has a non-finite entry")
    bg = t[:, 0]
    if ((bg != -1) & ((bg < 0) | (bg >= n_backgrounds) | (bg != np.floor(bg)))).any():
        raise ValueError(f"background index must be -1 or an integer in [0, {n_backgrounds})")
    if not np.isin(t[:, 1], (0, 1)).all() or not np.isin(t[:, 5], (NOISE_NONE, NOISE_GAUSS, NOISE_BLUR)).all():
        raise ValueError("chromatic must be 0 / 1 and noise 0 / 1 / 2")
    blur = t[:, 5] == NOISE_BLUR
    if not np.isin(t[blur, 7], BLUR_SIZES).all() or not np.isin(t[blur, 8], (0, 1)).all():
        raise ValueError(f"blur size must be one of {BLUR_SIZES} and blur axis 0 / 1")
    if (t[t[:, 5] == NOISE_GAUSS, 6] < 0).any():
        raise ValueError("sigma must be >= 0")


def draw_params(rng: np.random.RandomState, B: int, n_backgrounds: int, chromatic: bool = True, add_noise: bool = True,
                device="cuda", depth: bool = False):
    """Per-image scalars with the reference's formulas, drawn from `rng` in its call order: background index
    (minibatch.py:133, only when n_backgrounds > 0), d_h = (rand - 0.5) * 0.02 * 180, d_l / d_s = (rand - 0.5) * 0.2 * 256
    (blob.py:78-83), then add_noise's r < 0.9, var = rand * 0.3 * 256 or sizes[randint(6)], rand < 0.5 (blob.py:105-127).
    depth=True draws the depth blob's add_noise only (minibatch.py:193-194).  Returns (params [B, NUM_PARAMS] f64, keys [B]
    int64 holding the u64 Philox keys), both on `device`."""
    if B < 1 or n_backgrounds < 0:
        raise ValueError("need B >= 1 and n_backgrounds >= 0")
    table = np.zeros((B, NUM_PARAMS), np.float64)
    table[:, 0] = -1.0
    for b in range(B):
        row = table[b]
        if not depth:
            if n_backgrounds > 0:
                row[0] = rng.randint(n_backgrounds, size=1)[0]
            if chromatic:
                row[1] = 1.0
                row[2] = ((rng.rand(1) - 0.5) * 0.02 * 180)[0]
                row[3] = ((rng.rand(1) - 0.5) * 0.2 * 256)[0]
                row[4] = ((rng.rand(1) - 0.5) * 0.2 * 256)[0]
        if add_noise:
            _draw_noise(rng, row)
    validate_params(table, n_backgrounds)
    keys = rng.randint(0, 2 ** 63, size=B, dtype=np.int64)
    return torch.from_numpy(table).to(device), torch.from_numpy(keys).to(device)


def background_pool(backgrounds) -> torch.Tensor:
    """Stack backgrounds [H,W,3] u8 (already at the frame size: the reference's per-draw cv2.resize(INTER_LINEAR) is deterministic,
    so resizing once up front gives the same pixels) into the pool [N,H,W,3] u8 on the host; move it to the device once."""
    arrs = [np.ascontiguousarray(b) for b in backgrounds]
    if not arrs or any(a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape != arrs[0].shape for a in arrs):
        raise ValueError("backgrounds must be a non-empty list of [H,W,3] uint8 arrays of one size")
    return torch.from_numpy(np.stack(arrs))


def _common(params, keys, noise_field, B, H, W, dev):
    params = require_cuda("params", params, torch.float64, 2)
    keys = require_cuda("keys", keys, torch.int64, 1)
    if tuple(params.shape) != (B, NUM_PARAMS) or keys.numel() != B:
        raise ValueError(f"params must be [{B}, {NUM_PARAMS}] and keys [{B}]")
    if noise_field is not None:
        noise_field = require_cuda("noise_field", noise_field, torch.float64, 3)
        if tuple(noise_field.shape) != (B, H, W):
            raise ValueError(f"noise_field must be [{B}, {H}, {W}]")
    if params.device != dev or keys.device != dev or (noise_field is not None and noise_field.device != dev):
        raise ValueError("all tensors must be on one device")
    return params, keys, noise_field


def augment_color(rgba: torch.Tensor, backgrounds: torch.Tensor | None, params: torch.Tensor, keys: torch.Tensor,
                  noise_field: torch.Tensor | None = None, mean=PIXEL_MEANS) -> torch.Tensor:
    """rgba [B,H,W,4] u8 (or [B,H,W,3]: no alpha), backgrounds [N,H,W,3] u8 or None -> the colour blob [B,H,W,3] f32
    (pcnn_augment_color_fwd): composite, chromatic_transform, add_noise, - mean."""
    rgba = require_cuda("rgba", rgba, torch.uint8, 4)
    B, H, W, ch = rgba.shape
    if ch not in (3, 4):
        raise ValueError("rgba must have 3 or 4 channels")
    n_bg = 0
    if backgrounds is not None:
        backgrounds = require_cuda("backgrounds", backgrounds, torch.uint8, 4)
        if tuple(backgrounds.shape[1:]) != (H, W, 3) or backgrounds.device != rgba.device:
            raise ValueError(f"backgrounds must be [N, {H}, {W}, 3] on the images' device")
        n_bg = backgrounds.shape[0]
    params, keys, noise_field = _common(params, keys, noise_field, B, H, W, rgba.device)
    out = torch.empty((B, H, W, 3), dtype=torch.float32, device=rgba.device)
    m = (ctypes.c_double * 3)(*mean)
    check(lib().pcnn_augment_color_fwd(ptr(rgba), ch, ptr(backgrounds if n_bg else None), n_bg, ptr(params), ptr(keys),
                                       ptr(noise_field), B, H, W, m, ptr(out), stream()))
    return out


def depth_blob_train(depth: torch.Tensor, params: torch.Tensor, keys: torch.Tensor, noise_field: torch.Tensor | None = None,
                     mean=PIXEL_MEANS, return_max: bool = False):
    """depth [B,H,W] u16 (passed as torch.uint16) or f32 -> the training depth blob [B,H,W,3] f32 (pcnn_depth_blob_train_fwd):
    d / max(d) * 255 tiled x3, add_noise, - mean.  return_max=True also returns max(d) [B] f32."""
    if not isinstance(depth, torch.Tensor) or depth.dtype not in (torch.uint16, torch.float32):
        raise TypeError("depth must be a torch.uint16 or torch.float32 tensor")
    depth = require_cuda("depth", depth, depth.dtype, 3)
    B, H, W = depth.shape
    params, keys, noise_field = _common(params, keys, noise_field, B, H, W, depth.device)
    out = torch.empty((B, H, W, 3), dtype=torch.float32, device=depth.device)
    dmax = torch.empty((B,), dtype=torch.float32, device=depth.device)
    m = (ctypes.c_double * 3)(*mean)
    check(lib().pcnn_depth_blob_train_fwd(ptr(depth), int(depth.dtype == torch.uint16), ptr(params), ptr(keys), ptr(noise_field), B, H,
                                          W, m, ptr(dmax), ptr(out), stream()))
    return (out, dmax) if return_max else out
