"""Reference windows of the region proposal network, restated from lib/rpn_layer/generate_anchors.py (Faster R-CNN): for each
aspect ratio (outer loop) and each scale (inner loop), a box centred on the base window (0, 0, base_size - 1, base_size - 1),
in float64 as the reference computes them."""
from __future__ import annotations

import numpy as np


def _boxes_around(cx, cy, ws, hs):
    return np.stack([cx - 0.5 * (ws - 1), cy - 0.5 * (hs - 1), cx + 0.5 * (ws - 1), cy + 0.5 * (hs - 1)], axis=1)


def generate_anchors(base_size=16, ratios=(0.5, 1, 2), scales=(8, 16, 32)):
    """[len(ratios) * len(scales), 4] float64 (x1, y1, x2, y2)."""
    ratios = np.asarray(ratios, dtype=np.float64)
    scales = np.asarray(scales, dtype=np.float64)
    side = float(base_size)
    cx = cy = 0.5 * (side - 1)
    # the ratio windows keep the base area: width round(sqrt(area / r)), height round(width * r) (numpy round: half to even)
    ws = np.round(np.sqrt(side * side / ratios))
    hs = np.round(ws * ratios)
    out = [_boxes_around(cx, cy, w * scales, h * scales) for w, h in zip(ws, hs)]
    return np.concatenate(out, axis=0)
