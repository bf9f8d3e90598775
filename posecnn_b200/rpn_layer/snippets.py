"""Anchors of a feature map, restated from lib/rpn_layer/snippets.py::generate_anchors_pre."""
from __future__ import annotations

import numpy as np

from .generate_anchors import generate_anchors


def generate_anchors_pre(height, width, feat_stride, anchor_scales=(8, 16, 32), anchor_ratios=(0.5, 1, 2)):
    """The anchors of a height x width map at stride feat_stride: [height * width * A, 4] float32 in (h, w, a) order (a
    fastest), each base anchor shifted by (x * feat_stride, y * feat_stride); and their number as np.int32."""
    base = generate_anchors(ratios=np.array(anchor_ratios), scales=np.array(anchor_scales))
    ys, xs = np.meshgrid(np.arange(height) * feat_stride, np.arange(width) * feat_stride, indexing="ij")
    shifts = np.stack([xs.ravel(), ys.ravel(), xs.ravel(), ys.ravel()], axis=1)
    anchors = (shifts[:, None, :] + base[None, :, :]).reshape(-1, 4).astype(np.float32)
    return anchors, np.int32(anchors.shape[0])
