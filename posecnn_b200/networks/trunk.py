"""The VGG16 trunk conv1_1 .. conv5_3 that vgg16_convs and vgg16_det share (vgg16_convs.py:80-97, vgg16_det.py:51-68)."""
from __future__ import annotations

import torch

from .. import conv

PIXEL_MEANS = (102.9801, 115.9465, 122.7717)  # lib/fcn/config.py:242 (BGR)

VGG_CFG = [("conv1_1", 3, 64), ("conv1_2", 64, 64), "pool1", ("conv2_1", 64, 128), ("conv2_2", 128, 128), "pool2",
           ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), "pool3", ("conv4_1", 256, 512),
           ("conv4_2", 512, 512), ("conv4_3", 512, 512), "pool4", ("conv5_1", 512, 512), ("conv5_2", 512, 512),
           ("conv5_3", 512, 512)]


def trunk_shapes(sfx=""):
    """{`conv*{sfx}/weights`: HWIO, `conv*{sfx}/biases`: (Cout,)} of the 13 trunk layers."""
    shapes = {}
    for item in VGG_CFG:
        if isinstance(item, tuple):
            name, ci, co = item
            shapes[f"{name}{sfx}/weights"] = (3, 3, ci, co)
            shapes[f"{name}{sfx}/biases"] = (co,)
    return shapes


def conv_weights_to_tc(w: torch.Tensor) -> torch.Tensor:
    """A conv layer's HWIO weights -> the tensor-core layout its kernel reads (conv1_1: the im2col K order)."""
    return conv.conv1_1_weights_to_tc(w) if w.shape[2] == 3 else conv.hwio_to_tc(w)


def run_trunk(P, T, data, sfx=""):
    """13 x (conv3x3 + bias + ReLU), 4 x max-pool -> {"conv4_3", "conv5_3"} bf16.  P: f32 parameters, T: tensor-core weights
    (conv_weights_to_tc).  data: [B,H,W,3] u8 (BGR, mean subtracted on the fly) or f32 (already pre-processed), or [B,H,W] f32 = a
    RAW depth image (sensor units) whose blob clip(d / 2000, 0, 1) * 255 x3 - PIXEL_MEANS (lib/fcn/test.py:70-76) is formed in
    the conv1_1 loader."""
    if data.dim() == 3:
        x = conv.conv1_depth_fused(data, T[f"conv1_1{sfx}/weights"], P[f"conv1_1{sfx}/biases"], PIXEL_MEANS, True)
    else:
        mean = PIXEL_MEANS if data.dtype == torch.uint8 else None
        x = conv.conv1_fused(data, T[f"conv1_1{sfx}/weights"], P[f"conv1_1{sfx}/biases"], mean, True)
    feats = {}
    cfg = VGG_CFG[1:]
    i = 0
    while i < len(cfg):
        item = cfg[i]
        if isinstance(item, str):
            x = conv.maxpool2x2(x)
            i += 1
            continue
        name = item[0]
        fuse_pool = i + 1 < len(cfg) and isinstance(cfg[i + 1], str) and name not in ("conv4_3", "conv5_3")
        if fuse_pool:   # conv + ReLU + max-pool in one kernel (the un-pooled tensor is not needed downstream)
            x = conv.conv_pool_bf16(x, T[f"{name}{sfx}/weights"], P[f"{name}{sfx}/biases"], 3, True)
            i += 2
            continue
        x = conv.conv_bf16(x, T[f"{name}{sfx}/weights"], P[f"{name}{sfx}/biases"], 3, True)
        if name in ("conv4_3", "conv5_3"):
            feats[name] = x
        i += 1
    return feats
