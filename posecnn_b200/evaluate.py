"""Evaluation of the test-time records on the device (csrc/evaluate.cu, DESIGN.md §14): the segmentation confusion matrix and
the pose accuracy the reference's scorer reports (lib/fcn/test.py:1432, 1466 -> lib/datasets/lov.py:397-680,
linemod.py:626-760, lib/utils/pose_error.py).

`Evaluator` keeps its whole state in one int64 device tensor (histogram, counts and the argument-error counters), so scoring
batches never synchronises with the host and can be captured in a CUDA graph; `summary()` makes the only device-to-host copy.
Two-class models (LINEMOD, the per-object YCB models) score in their own numbering: pass the label map and gt rows of
single_class.single_class_view and the two-row tables, as linemod.py:648-670 remaps them.
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import check, lib, ptr, require_cuda, stream

# lov.py:601: the classes scored with ADD-S (adi) in the YCB-Video class numbering: 024_bowl, 036_wood_block, 061_foam_brick.
# Not synth.LOV_SYMMETRY (the training table of lov.py:38 marks only 16 and 21).
LOV_EVAL_SYMMETRIC = np.zeros(22, np.float32)
LOV_EVAL_SYMMETRIC[[13, 16, 21]] = 1.0

MAX_POSE_SETS = 4
MAX_GT_ROWS = 4096


def gt_rows_from_meta(batch, cls_indexes, poses_3x4xn) -> np.ndarray:
    """[n,14] float32 gt rows (image, class, [R | t] row-major) from a frame's meta data: cls_indexes [n] and poses [3,4,n]
    (a single [3,4] pose is one object, lov.py:572-573).  Host arrays; the dataset loader is the caller's."""
    poses = np.asarray(poses_3x4xn, np.float64)
    if poses.ndim == 2:
        poses = poses.reshape(3, 4, 1)
    cls = np.asarray(cls_indexes).reshape(-1)
    if poses.shape[:2] != (3, 4) or poses.shape[2] != cls.shape[0]:
        raise ValueError("poses must be [3,4,n] with one class index per pose")
    rows = np.zeros((cls.shape[0], 14), np.float32)
    rows[:, 0] = batch
    rows[:, 1] = cls
    rows[:, 2:] = poses.transpose(2, 0, 1).reshape(-1, 12)
    return rows


def gt_rows_from_pose_blob(poses13: torch.Tensor) -> torch.Tensor:
    """[n,14] gt rows on the device from the data layer's pose blob [n,13] (image, class, box, quaternion, translation): R by
    quat2mat, in fp64 rounded to fp32 (the conversion the estimates get)."""
    blob = require_cuda("poses13", poses13, torch.float32, 2)
    if blob.shape[1] != 13:
        raise ValueError("the pose blob must be [n,13]")
    rows = torch.empty((blob.shape[0], 14), dtype=torch.float32, device=blob.device)
    check(lib().pcnn_eval_gt_rows_from_blob(ptr(blob), blob.shape[0], ptr(rows), stream()))
    return rows


class Evaluator:
    """Accumulates the reference's evaluation figures over batches on the device.

    num_classes C (2 <= C <= 128), points [C,P,3] (P <= 4096), extents [C,3], symmetric [C] (> 0: ADD-S, e.g. LOV_EVAL_SYMMETRIC),
    threshold [C] (default 0.1 ||extents[c]||, lov.py:539-541), flip_z [C] (> 0: LINEMOD's eggbox rule, default none), pose_sets:
    names of the record sets scored (e.g. ("poses", "poses_refined", "poses_icp"), and "poses_rgb" for the colour-only records of
    a VERTEX_REG_3D network, scored in their own add_poses call with their own rois)."""

    def __init__(self, num_classes, points, extents, symmetric, threshold=None, flip_z=None, pose_sets=("poses",), device="cuda"):
        C = int(num_classes)
        if not 2 <= C <= 128:
            raise ValueError(f"num_classes = {C} (2 <= C <= 128)")
        self.num_classes = C
        self.device = torch.device(device)
        f32 = lambda a, n: torch.as_tensor(np.ascontiguousarray(np.asarray(a, np.float32).reshape(n)), device=self.device)
        ext = np.asarray(extents, np.float32).reshape(C, 3)
        self.points = torch.as_tensor(np.asarray(points, np.float32), device=self.device).contiguous() \
            if not isinstance(points, torch.Tensor) else points.to(self.device, torch.float32).contiguous()
        if self.points.dim() != 3 or self.points.shape[0] != C or self.points.shape[2] != 3:
            raise ValueError("points must be [C,P,3]")
        if threshold is None:
            threshold = [0.1 * np.linalg.norm(e) for e in ext]          # lov.py:541, stored as float32
        self.symmetric = f32(symmetric, C)
        self.threshold = f32(threshold, C)
        self.flip_z = f32(np.zeros(C) if flip_z is None else flip_z, C)
        self.pose_sets = tuple(pose_sets)
        if not self.pose_sets or len(set(self.pose_sets)) != len(self.pose_sets):
            raise ValueError("pose_sets must be distinct names")
        S = len(self.pose_sets)
        # one int64 tensor: hist [C*C] | status [2] (bad predictions, bad gt rows / row counts) | counts [S,3,C]
        self.state = torch.zeros(C * C + 2 + S * 3 * C, dtype=torch.int64, device=self.device)
        self.hist = self.state[:C * C].view(C, C)
        self.status = self.state[C * C:C * C + 2]
        self.counts = self.state[C * C + 2:].view(S, 3, C)

    def add_labels(self, gt_label: torch.Tensor, label: torch.Tensor):
        """gt_label, label [B,H,W] int32 (gt -1 = not annotated: skipped).  Adds the batch's confusion matrix."""
        g = require_cuda("gt_label", gt_label, torch.int32)
        p = require_cuda("label", label, torch.int32)
        if g.shape != p.shape:
            raise ValueError("gt_label and label must have the same shape")
        check(lib().pcnn_eval_confusion(ptr(g), ptr(p), g.numel(), self.num_classes, ptr(self.hist), ptr(self.status), stream()))

    def add_poses(self, gt_rows: torch.Tensor, rois: torch.Tensor, poses: dict, num_rows: torch.Tensor | None, meta_data: torch.Tensor,
                  batch_offset: int = 0) -> dict:
        """Scores one batch: gt_rows [n,14] f32 (gt_rows_from_meta / gt_rows_from_pose_blob), rois [cap,>=2] (image, class, ...),
        poses {set name: [cap,7]} (1 to 4 of the evaluator's sets), num_rows device int32 [1] or None (= cap), meta_data [B,...]
        f32 (K in [0:9]); images are numbered from batch_offset.  Returns the per-pair rows on the device: pairs [n*cap,2] int32
        (gt index, record row), errors [S,n*cap,4] f64 (re deg, te, ADD or ADD-S, reproj px) and flags [S,n*cap] int32 (bit0
        under the threshold, bit1 under 5 px, bit2 eggbox flip), valid for the first num_pairs [1] int32 rows; sets: the names."""
        if not 1 <= len(poses) <= MAX_POSE_SETS:
            raise ValueError("poses must hold 1 to 4 pose sets")
        idx = []
        for name in poses:
            if name not in self.pose_sets:
                raise KeyError(f"pose set {name!r} is not one of {self.pose_sets}")
            idx.append(self.pose_sets.index(name))
        g = require_cuda("gt_rows", gt_rows, torch.float32, 2)
        r = require_cuda("rois", rois, torch.float32, 2)
        cap = r.shape[0]
        if g.shape[1] != 14 or g.shape[0] > MAX_GT_ROWS:
            raise ValueError(f"gt_rows must be [n,14] with n <= {MAX_GT_ROWS}")
        P = [require_cuda(f"poses[{k!r}]", v, torch.float32, 2) for k, v in poses.items()]
        if any(tuple(p.shape) != (cap, 7) for p in P):
            raise ValueError("every pose set must be [cap,7] like rois")
        meta = require_cuda("meta_data", meta_data, torch.float32)
        meta = meta.reshape(meta.shape[0], -1)
        nr = None if num_rows is None else require_cuda("num_rows", num_rows, torch.int32).reshape(-1)
        n, S = g.shape[0], len(P)
        dev = self.device
        pairs = torch.empty((n * cap, 2), dtype=torch.int32, device=dev)
        errors = torch.empty((S, n * cap, 4), dtype=torch.float64, device=dev)
        flags = torch.empty((S, n * cap), dtype=torch.int32, device=dev)
        num_pairs = torch.empty(1, dtype=torch.int32, device=dev)
        counts = torch.zeros((S, 3, self.num_classes), dtype=torch.int64, device=dev)
        pp = [ptr(p) for p in P] + [None] * (MAX_POSE_SETS - S)
        check(lib().pcnn_eval_pose_errors(ptr(g), n, ptr(r), r.shape[1], cap, ptr(nr), *pp, S, ptr(meta), meta.shape[1], meta.shape[0],
                                          int(batch_offset), ptr(self.points), self.num_classes, self.points.shape[1],
                                          ptr(self.symmetric), ptr(self.threshold), ptr(self.flip_z), ptr(pairs), ptr(errors),
                                          ptr(flags), ptr(num_pairs), ptr(counts), ptr(self.status), stream()))
        for k, i in enumerate(idx):
            self.counts[i] += counts[k]
        return dict(pairs=pairs, errors=errors, flags=flags, num_pairs=num_pairs, sets=list(poses))

    def merge(self, other: "Evaluator"):
        """Adds another evaluator's state (the same classes and pose sets), e.g. one scoring another shard of the images."""
        if other.num_classes != self.num_classes or other.pose_sets != self.pose_sets:
            raise ValueError("merge needs evaluators of the same classes and pose sets")
        self.state += other.state.to(self.device)

    def all_reduce(self):
        """Sums the state over the default torch.distributed process group (every rank holds the total afterwards)."""
        import torch.distributed as dist
        dist.all_reduce(self.state, op=dist.ReduceOp.SUM)

    def summary(self) -> dict:
        """The reference's figures (lov.py:645-680): overall_accuracy, mean_accuracy (nanmean of the per-class accuracy),
        per_class_iu [C], mean_iu (nanmean), fwavacc, hist [C,C], and per pose set count_all / count_correct / count_pixel [C] with
        accuracy = count_correct / count_all and accuracy_pixel = count_pixel / count_all (NaN where count_all is 0).  Raises when
        a predicted label was outside [0, C) or a gt row's image was outside the scored batch."""
        st = self.state.cpu().numpy()
        C = self.num_classes
        bad_pred, bad_gt = int(st[C * C]), int(st[C * C + 1])
        if bad_pred or bad_gt:
            raise ValueError(f"evaluation inputs out of range: {bad_pred} predicted labels outside [0, {C}), {bad_gt} gt rows with an "
                             "image outside the batch or row counts outside [0, cap]")
        hist = st[:C * C].reshape(C, C).astype(np.float64)
        counts = st[C * C + 2:].reshape(len(self.pose_sets), 3, C)
        with np.errstate(divide="ignore", invalid="ignore"):
            diag = np.diag(hist)
            acc_cls = diag / hist.sum(1)
            iu = diag / (hist.sum(1) + hist.sum(0) - diag)
            freq = hist.sum(1) / hist.sum()
            out = dict(overall_accuracy=diag.sum() / hist.sum(), mean_accuracy=_nanmean(acc_cls), per_class_iu=iu,
                       mean_iu=_nanmean(iu), fwavacc=(freq[freq > 0] * iu[freq > 0]).sum(), hist=hist.astype(np.int64), poses={})
            for s, name in enumerate(self.pose_sets):
                a, c, p = counts[s]
                out["poses"][name] = dict(count_all=a, count_correct=c, count_pixel=p, accuracy=c / a, accuracy_pixel=p / a)
        return out


def _nanmean(x):
    return float(np.nanmean(x)) if np.isfinite(x).any() else float("nan")
