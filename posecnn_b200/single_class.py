"""The single-object (two-class) view of a multi-object frame: how the reference trains and tests its num_classes = 2 models
(the LINEMOD models, experiments/cfgs/linemod_*.yml, and the per-object YCB models lov_color_<object>.yml / ycb_color_*.yml).

Its loader (lib/gt_synthesize_layer/minibatch.py:355-367) and its test driver (lib/fcn/test.py:1284-1294) rewrite the annotation
of a frame for the object `cls_index` of the dataset's class list:
    label          label == cls_index -> 1, every other class -> 0
    poses / centre only the rows of cls_index are kept, with class 1
and the dataset object supplies two-row tables (lib/datasets/linemod.py:30-51, 167-195): classes (background, object),
extents[1] = the object's extents, symmetry = [0, symmetry of the object], points[1] = the object's model points.
The inverse (test.py:1409-1414, before the ICP refinement) lives in utils/results.py: to_dataset_classes.
"""
from __future__ import annotations

import torch


def single_class_view(cls_index: int, gt_label_2d: torch.Tensor, centers: torch.Tensor, gt_poses: torch.Tensor, extents: torch.Tensor,
                      points: torch.Tensor, symmetry: torch.Tensor) -> dict:
    """The two-class inputs of Trainer.step / vgg16_convs.forward from the dataset-wide ones, on the tensors' own device.

    gt_label_2d [B,H,W] int32    -> label == cls_index: 1, other classes 0; -1 (ignored / unannotated pixels, an adapt batch)
                                    stays -1 (the reference's label images have no such value)
    centers     [B,C,3]          -> [B,2,3]: row 1 = the object's projected centre and depth, row 0 zero
    gt_poses    [N,13]           -> the rows [b, cls, box, quaternion, translation] of cls_index, with class 1, in their order
                                    (a data-dependent row count: one device-to-host read)
    extents     [C,3]            -> [2,3]: row 0 zero, row 1 = extents[cls_index] (a table with the background row 0, lov.py:168; the
                                    same row as linemod.py's extents_all[cls_index - 1] of extents.txt)
    points      [C,P,3]          -> [2,P,3]: row 0 zero, row 1 = the object's points
    symmetry    [C]              -> [0, symmetry[cls_index]]
    The label remap is one element-wise pass on the device; everything else is a row selection.  The object-coordinate map of a
    VERTEX_REG_3D batch (Trainer.step's vertmap [B,H,W,3]) needs no view: it is per pixel, not indexed by class, and the two-row
    extents above already scale the object's coordinates."""
    c = int(cls_index)
    if not 1 <= c < centers.shape[1]:
        raise ValueError(f"cls_index must be a foreground class of the {centers.shape[1]}-class tables (got {c})")
    lab = gt_label_2d
    label = torch.where(lab < 0, lab, (lab == c).to(lab.dtype))
    cen = centers.new_zeros((centers.shape[0], 2, 3))
    cen[:, 1] = centers[:, c]
    poses = gt_poses.reshape(-1, 13)
    poses = poses[poses[:, 1] == c].clone()
    poses[:, 1] = 1.0
    ext = extents.new_zeros((2, 3))
    ext[1] = extents[c]
    pts = points.new_zeros((2,) + tuple(points.shape[1:]))
    pts[1] = points[c]
    sym = symmetry.new_zeros((2,))
    sym[1] = symmetry[c]
    return dict(label=label.contiguous(), centers=cen, gt_poses=poses.contiguous(), extents=ext, points=pts, symmetry=sym)
