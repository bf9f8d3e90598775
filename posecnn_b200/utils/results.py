"""Result records handed to pose refinement and to the evaluation scripts (SURVEY.md §8(f) rank 4).

The reference keeps one dictionary per image (`lib/fcn/test.py:1415-1423`), feeds `rois` / `poses` to the ICP refiner
(`synthesizer.icp_python`, `test.py:1327-1351`: 7 camera parameters + ROI rows + pose rows) and writes the dictionary
with `scipy.io.savemat(..., do_compression=True)` (`lib/datasets/lov.py:431-438`).  Row layouts are the ones the
network emits: rois `[batch, cls, x1, y1, x2, y2, score]`, poses `[qw, qx, qy, qz, tx, ty, tz]`.
"""
from __future__ import annotations

import numpy as np

ROI_COLUMNS = ("batch", "cls", "x1", "y1", "x2", "y2", "score")
POSE_COLUMNS = ("qw", "qx", "qy", "qz", "tx", "ty", "tz")
ZNEAR, ZFAR = 0.25, 6.0                       # test.py:1322-1323
ICP_ERROR_THRESHOLD = 0.01                    # test.py:1326


def split_detections(records, batch: int):
    """Gathered post-NMS records [rows, 15] (posecnn_b200.parallel.pack_detections: roi | pose | valid) -> list of
    (rois [n,7], poses [n,7]) per GLOBAL image index, rows in processing (score) order."""
    rec = np.asarray(records, dtype=np.float32)
    rec = rec[rec[:, 14] > 0]
    out = []
    for b in range(batch):
        sel = rec[rec[:, 0] == b]
        out.append((sel[:, 0:7].copy(), sel[:, 7:14].copy()))
    return out


def icp_parameters(intrinsic_matrix, factor_depth, im_scale=1.0):
    """The 7-vector `parameters` of test.py:1338-1345: fx, fy, px, py (scaled), znear, zfar, depth factor."""
    K = np.asarray(intrinsic_matrix, dtype=np.float64)
    return np.array([K[0, 0] * im_scale, K[1, 1] * im_scale, K[0, 2] * im_scale, K[1, 2] * im_scale, ZNEAR, ZFAR, factor_depth],
                    dtype=np.float32)


def segmentation_record(labels, rois, poses, poses_refined=None, poses_icp=None):
    """The per-image dictionary of test.py:1415-1419 (VERTEX_REG_2D): refined / ICP poses default to zeros [n,7]
    (test.py:1324-1325); posecnn_b200.pose_refine fills them."""
    rois = np.ascontiguousarray(rois, dtype=np.float32).reshape(-1, 7)
    poses = np.ascontiguousarray(poses, dtype=np.float32).reshape(-1, 7)
    if rois.shape[0] != poses.shape[0]:
        raise ValueError("rois and poses must have the same number of rows")
    z = lambda a: np.zeros((poses.shape[0], 7), np.float32) if a is None else np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 7)
    return {"labels": np.ascontiguousarray(labels, dtype=np.int32), "rois": rois, "poses": poses, "poses_refined": z(poses_refined),
            "poses_icp": z(poses_icp)}


def to_dataset_classes(labels, rois, cls_index):
    """A two-class model's output in the dataset's class numbering, as test.py:1409-1414 hands it to the ICP refiner: every
    label > 0 becomes cls_index and every ROI row's class column becomes cls_index (copies; the inputs are not changed).
    The forward direction is posecnn_b200.single_class.single_class_view."""
    labels = np.array(labels, dtype=np.int32, copy=True)
    labels[labels > 0] = int(cls_index)
    rois = np.array(rois, dtype=np.float32, copy=True).reshape(-1, 7)
    rois[:, 1] = cls_index
    return labels, rois


def save_mat(filename, record):
    """lov.py:431-438: `scipy.io.savemat(filename, results, do_compression=True)`."""
    import scipy.io
    scipy.io.savemat(filename, record, do_compression=True)
