"""Generate tests/golden/vertex_targets_3d.npz by EXECUTING THE REFERENCE'S OWN VERTEX_REG_3D target code:
`_generate_vertex_targets` (single-instance branch) and `_scale_vertmap` of lib/gt_synthesize_layer/minibatch.py:543-616, with
cfg.TRAIN.VERTEX_REG_3D = True and VERTEX_REG_2D = False (the linemod_*_3d.yml / lov_color_3d.yml configurations).  The module is
Python 2 and cannot be imported, so the two functions are cut out of the file unmodified (only de-indented) and exec'd with the
names they read (np, cfg, xrange = range).

Precision: the arithmetic is numpy's on float32 operands (extents and vertmap are float32 arrays, the blobs float32).  This file
relies on numpy 2 (NEP 50): vmin, vmax, a and b are float32 scalars and a * v + b runs as two rounded float32 operations.  numpy 1's
value-based casting makes a = 1.0 / (vmax - vmin) a float64 scalar instead, which is cast to float32 before the float32 array
multiply; a float64 quotient of float32 operands rounded to float32 equals the float32 quotient, and b = (e / 2) / e = 0.5 exactly in
both, so numpy 1 writes the same bits.  main() checks the float32 scalars and that the result equals the float32 recipe.

    python tests/golden/make_golden_vertex_3d.py        # needs the reference's sources; the .npz is committed

Cases: several classes per image; a class with pixels that is not listed in the frame (no target, weight 0); a listed class
with no pixels; a zero-extent axis and a negative one (a = b = 0 there); ignored pixels (label -1); full-mantissa coordinates,
including values outside the extent box and on its faces.
"""
import os
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference/lib"
B, H, W, C = 2, 24, 32, 6
W_INSIDE = 10.0


def cut(path, first, last):
    """The lines from the first one starting with `first` to the next one starting with `last`, both stripped of indentation."""
    src = open(path).read().splitlines()
    s = next(i for i, l in enumerate(src) if l.strip().startswith(first))
    e = next(i for i in range(s, len(src)) if src[i].strip().startswith(last))
    return textwrap.dedent("\n".join(src[s:e + 1]))


def inputs():
    """label [B,H,W] int32, vertmap [B,H,W,3] f32, extents [C,3] f32 (row 0 = background), cls_indexes per image (the listed
    classes, in the frame's order)."""
    rng = np.random.default_rng(23)
    ext = rng.uniform(0.04, 0.3, (C, 3)).astype(np.float32)
    ext[0] = 0.0
    ext[2, 1] = 0.0                                   # zero-extent axis: a = b = 0
    ext[5, 2] = -0.07                                 # negative axis: vmax - vmin < 0, a = b = 0
    label = np.zeros((B, H, W), np.int32)
    boxes = [[(1, 2, 3, 10, 14), (2, 12, 2, 22, 12), (3, 4, 16, 16, 28), (1, 18, 18, 23, 30)],   # image 0: classes 1, 2, 3
             [(5, 1, 1, 12, 20), (1, 10, 14, 22, 31), (4, 20, 0, 24, 6)]]                      # image 1: classes 5, 1, 4
    for b, bx in enumerate(boxes):
        for (c, y0, x0, y1, x1) in bx:
            label[b, y0:y1, x0:x1] = c
    label[0, 5, 5:9] = -1                             # ignored pixels
    cls_indexes = [np.array([2, 1, 4], np.float64),   # class 3 has pixels but is not listed; class 4 is listed without pixels
                   np.array([5, 1, 3], np.float64)]   # class 4 has pixels but is not listed; class 3 is listed without pixels
    # object coordinates across (and beyond) each class's box, full float32 mantissas; a few exactly on the faces
    scale = np.maximum(np.abs(ext[np.clip(label, 0, None)]), 0.05)
    vertmap = (rng.uniform(-0.65, 0.65, (B, H, W, 3)) * scale).astype(np.float32)
    faces = np.nonzero(label == 1)
    for k in range(3):
        vertmap[faces[0][k], faces[1][k], faces[2][k], k] = ext[1, k] / np.float32(2)
        vertmap[faces[0][-1 - k], faces[1][-1 - k], faces[2][-1 - k], k] = -ext[1, k] / np.float32(2)
    return label, vertmap, ext, cls_indexes


def float32_recipe(label, vertmap, ext, cls_indexes):
    """The target as the float32 recipe states it (the check that the reference's arithmetic is that recipe)."""
    t = np.zeros((B, H, W, 3 * C), np.float32)
    for b in range(B):
        for c in range(1, C):
            m = label[b] == c
            if not m.any() or c not in cls_indexes[b]:
                continue
            for k in range(3):
                vmin, vmax = -ext[c, k] / np.float32(2), ext[c, k] / np.float32(2)
                span = vmax - vmin
                a = np.float32(1) / span if span > 0 else np.float32(0)
                bb = (np.float32(-1) * vmin) / span if span > 0 else np.float32(0)
                t[b][m, 3 * c + k] = (vertmap[b][m, k] * a).astype(np.float32) + bb
    return t


def main():
    mb = os.path.join(REF, "gt_synthesize_layer", "minibatch.py")
    gen = cut(mb, "def _generate_vertex_targets(", "return vertex_targets, vertex_weights")
    scale = cut(mb, "def _scale_vertmap(", "return vertmap[index[0], index[1], :]")
    cfg = types.SimpleNamespace(TRAIN=types.SimpleNamespace(VERTEX_REG_2D=False, VERTEX_REG_3D=True, VERTEX_W_INSIDE=W_INSIDE))
    ns = dict(np=np, cfg=cfg, xrange=range)
    exec(scale, ns)
    exec(gen, ns)
    label, vertmap, ext, cls_indexes = inputs()
    e = ext[1]
    vmin = -e[0] / 2
    assert isinstance(vmin, np.float32) and isinstance(1.0 / (e[0] / 2 - vmin), np.float32), "numpy 2 (NEP 50) scalar rules expected"
    targets = np.zeros((B, H, W, 3 * C), np.float32)
    weights = np.zeros((B, H, W, 3 * C), np.float32)
    for b in range(B):
        vm = vertmap[b].copy()                        # _scale_vertmap rewrites its argument in place
        targets[b], weights[b] = ns["_generate_vertex_targets"](label[b], cls_indexes[b], None, None, C, vm, ext, [], 0, None,
                                                                targets[b], weights[b])
    assert np.array_equal(targets.view(np.int32), float32_recipe(label, vertmap, ext, cls_indexes).view(np.int32))
    out = dict(label=label, vertmap=vertmap, extents=ext, targets=targets, weights=weights, w_inside=np.float32(W_INSIDE),
               **{f"cls_indexes{b}": cls_indexes[b] for b in range(B)})
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "vertex_targets_3d.npz"), **out)
    print("weighted pixels per image:", [(weights[b, ..., ::3] > 0).sum() for b in range(B)])


if __name__ == "__main__":
    main()
