"""Generate tests/golden/det_post.npz by running the REFERENCE'S OWN post-processing of the detection network:
lib/utils/bbox_transform.py (bbox_transform_inv, clip_boxes), and compute_translations / distance_objective of
lib/fcn/test.py with scipy's minimize.  test.py is a Python 2 module, so the source text of those two functions is extracted
and executed on its own.  quat2mat is the stub make_golden_eval.py uses (tests/eval_ref.quat2mat: transforms3d's formula on
float64), and nms is Fast R-CNN's lib/nms/py_cpu_nms.py: the `utils.nms.nms` test.py:18 binds reads seven columns and raises
IndexError on the five-column cls_dets of test.py:1599.  im_detect_single_frame's tail (test.py:1731-1746) and the class
loop (test.py:1589-1616) are restated around those calls, one image at a time, with im_scale = 1.

The inputs are seeded and tie-free at every class maximum.  At C = 22 and C = 2 they cover classes with nothing above 0.02,
boxes clipped to zero width, full-image boxes, tiny boxes (large depth), a zero quaternion and searches that stop at the
200-evaluation cap.  Every objective evaluation of every search is recorded (its z and value), as are nit and nfev.

    python tests/golden/make_golden_det_post.py          # needs /root/reference; the .npz is committed
"""
import os
import re
import sys

import numpy as np
from scipy.optimize import minimize

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF_LIB = "/root/reference/lib"
sys.path.insert(0, ROOT)

from posecnn_b200 import synth  # noqa: E402
from tests import eval_ref  # noqa: E402

F = np.float32
IM_H, IM_W = 480, 640
CASES = (("lov", 22, 2, 60, 400), ("linemod", 2, 6, 40, 1000))   # (tag, C, B, rows per image, points per class)


def make_case(tag, C, B, N, P, seed):
    """Seeded network outputs of B images with N proposal rows each (num_rois <= N), and the special records."""
    rng = np.random.default_rng(seed)
    x1 = rng.uniform(0, IM_W - 60, (B * N, 1)); y1 = rng.uniform(0, IM_H - 60, (B * N, 1))
    wh = rng.uniform(8, 200, (B * N, 2))
    rois = np.hstack([np.repeat(np.arange(B), N)[:, None], x1, y1, np.minimum(x1 + wh[:, :1], IM_W - 1),
                      np.minimum(y1 + wh[:, 1:], IM_H - 1)]).astype(F)
    logits = rng.normal(0, 2.0, (B * N, C))
    logits[:, 0] += 1.5
    prob = np.exp(logits) / np.exp(logits).sum(1, keepdims=True)
    cls_prob = prob.astype(F)
    bbox_pred = rng.normal(0, 1.0, (B * N, 4 * C)).astype(F)
    poses_tanh = np.tanh(rng.normal(0, 0.8, (B * N, 4 * C))).astype(F)
    num_rois = np.array([N - 3 * b for b in range(B)], np.int32)
    # image 0: class 1 has nothing above 0.02 (at C = 2: image 1 instead, so image 0 keeps its record)
    empty_img = 1 if C == 2 else 0
    assert C > 6 or B >= 6
    cls_prob[empty_img * N:(empty_img + 1) * N, 1] = rng.uniform(0, 0.02, N).astype(F)
    specials = []

    def plant(b, j, roi, deltas, q=None, score=F(1.0)):
        """Row 5 + len(specials) of image b becomes class j's top-scoring row with this box, deltas and quaternion."""
        r = b * N + 5 + len(specials)
        rois[r, 1:] = roi
        bbox_pred[r, 4 * j:4 * j + 4] = deltas
        if q is not None:
            poses_tanh[r, 4 * j:4 * j + 4] = q
        cls_prob[r, j] = score
        specials.append((b, j, r))

    K = synth.intrinsics(IM_H, IM_W)
    cx, cy = F(K[0, 2]) - F(0.5), F(K[1, 2]) - F(0.5)
    # (image, class) of each special record: a zero-size box at the principal point, whose search stops at the cap; x pushed
    # past the right edge (clipped to zero width at W - 1); the full image; a tiny box (large depth); a zero quaternion; a box
    # clipped to the corner (0, 0)
    at = dict(cap=(0, 6), clip=(0, 21), full=(1, 2), tiny=(0, 3), zero_q=(1, 4), corner=(1, 5)) if C > 2 else \
        dict(cap=(0, 1), clip=(2, 1), full=(3, 1), tiny=(4, 1), zero_q=(5, 1))
    plant(*at["cap"], (cx, cy, cx, cy), (0.0, 0.0, -1000.0, -1000.0))
    plant(*at["clip"], (500, 200, 560, 260), (60.0, 0.0, 0.0, 0.0))
    plant(*at["full"], (0, 0, IM_W - 1, IM_H - 1), (0.0, 0.0, 0.0, 0.0))
    plant(*at["tiny"], (320, 240, 323, 243), (0.0, 0.0, -12.0, -12.0))
    plant(*at["zero_q"], (100, 100, 180, 160), (0.1, -0.2, 0.3, 0.1), q=(0, 0, 0, 0))
    if "corner" in at:
        plant(*at["corner"], (10, 10, 60, 60), (-60.0, -60.0, 0.0, 0.0))
    for b in range(B):                                  # tie-free at every class maximum
        s = cls_prob[b * N:b * N + num_rois[b]]
        for j in range(1, C):
            top = s[:, j].max()
            assert top <= 0.02 or (s[:, j] == top).sum() == 1, (b, j)
    meta = np.stack([synth.make_meta(K)] * B).astype(F)
    meta[1, 2] += F(3.5)                                                                    # a second camera centre
    points = synth.make_model_points(C, P, seed=seed)
    return dict(cls_prob=cls_prob, bbox_pred=bbox_pred, poses_tanh=poses_tanh, rois=rois, num_rois=num_rois,
                meta=meta, points=points, im_hw=np.array([IM_H, IM_W], np.int32), specials=np.array(specials, np.int32))


def load_reference():
    sys.path.insert(0, REF_LIB)
    from nms.py_cpu_nms import py_cpu_nms
    from utils.bbox_transform import bbox_transform_inv, clip_boxes
    with open(os.path.join(REF_LIB, "fcn", "test.py")) as f:
        text = f.read()
    src = ""
    for name in ("compute_translations", "distance_objective"):
        m = re.search(rf"^def {name}\(.*?(?=^\S)", text, flags=re.S | re.M)
        src += m.group(0) + "\n"
    ns = dict(np=np, xrange=range, minimize=minimize, quat2mat=eval_ref.quat2mat)
    exec(compile(src, "lib/fcn/test.py", "exec"), ns)
    return bbox_transform_inv, clip_boxes, py_cpu_nms, ns


def reference_records(case, ref):
    """test.py:1589-1616 and 1731-1746 per image around the reference's functions; every objective call recorded."""
    bbox_transform_inv, clip_boxes, nms, ns = ref
    objective = ns["distance_objective"]
    calls, results = [], []

    def logged(x, *args):
        f = objective(x, *args)
        calls[-1].append((float(np.asarray(x).ravel()[0]), float(f)))
        return f

    def logged_minimize(*args, **kw):
        calls.append([])
        r = minimize(*args, **kw)
        results.append((int(r.nit), int(r.nfev), float(np.asarray(r.x).ravel()[0])))
        return r

    ns["distance_objective"], ns["minimize"] = logged, logged_minimize
    B, N = case["num_rois"].shape[0], case["rois"].shape[0] // case["num_rois"].shape[0]
    C = case["cls_prob"].shape[1]
    out_dets, out_poses = [], []
    for b in range(B):
        n = int(case["num_rois"][b])
        scores = case["cls_prob"][b * N:b * N + n].copy()
        bbox_pred = case["bbox_pred"][b * N:b * N + n].copy()
        rois = case["rois"][b * N:b * N + n].copy()
        poses = case["poses_tanh"][b * N:b * N + n].copy()
        stds = np.tile(np.array((0.1, 0.1, 0.2, 0.2)), C)                                 # test.py:1731-1734
        means = np.tile(np.array((0.0, 0.0, 0.0, 0.0)), C)
        bbox_pred *= stds
        bbox_pred += means
        boxes = rois[:, 1:5] / 1.0                                                         # test.py:1736, im_scale = 1
        pred_boxes = clip_boxes(bbox_transform_inv(boxes, bbox_pred), (IM_H, IM_W, 3))     # test.py:1742-1743
        all_dets = np.zeros((0, 6), dtype=np.float32)                                      # test.py:1590-1614
        all_poses = np.zeros((0, 7), dtype=np.float32)
        for j in range(1, C):
            inds = np.where(scores[:, j] > 0.02)[0]
            cls_scores = scores[inds, j]
            cls_boxes = pred_boxes[inds, j * 4:(j + 1) * 4]
            cls_poses = poses[inds, j * 4:(j + 1) * 4]
            cls_dets = np.hstack((cls_boxes, cls_scores[:, np.newaxis])).astype(np.float32, copy=False)
            keep = nms(cls_dets, 0.3)
            if len(keep) > 1:
                keep = [keep[0]]
            cls_dets = cls_dets[keep, :]
            cls_poses = cls_poses[keep, :]
            num = cls_dets.shape[0]
            if num > 0:
                cls_dets = np.hstack((j * np.ones((num, 1), dtype=np.float32), cls_dets))
                all_dets = np.vstack((all_dets, cls_dets))
                all_poses = np.vstack((all_poses, np.hstack((cls_poses, np.zeros((num, 3), dtype=np.float32)))))
        K = case["meta"][b, :9].astype(np.float64).reshape(3, 3)                           # the f32 meta data's values
        all_poses = ns["compute_translations"](all_dets, all_poses, case["points"], K)    # test.py:1616
        out_dets.append(np.hstack([np.full((all_dets.shape[0], 1), b, np.float32), all_dets]))
        out_poses.append(all_poses)
    dets, poses = np.vstack(out_dets), np.vstack(out_poses)
    xs = np.full((len(calls), 200), np.nan)
    fs = np.full((len(calls), 200), np.nan)
    for i, c in enumerate(calls):
        xs[i, :len(c)] = [v[0] for v in c]
        fs[i, :len(c)] = [v[1] for v in c]
    return dict(dets=dets, poses=poses, evals=np.array([len(c) for c in calls], np.int32), xs=xs, fs=fs,
                nit_nfev=np.array([r[:2] for r in results], np.int32), z=np.array([r[2] for r in results]))


def main():
    ref = load_reference()
    out = {}
    for k, (tag, C, B, N, P) in enumerate(CASES):
        case = make_case(tag, C, B, N, P, seed=500 + k)
        for name, v in case.items():
            out[f"{tag}_{name}"] = v
        for name, v in reference_records(case, ref).items():
            out[f"{tag}_ref_{name}"] = v
        nf = out[f"{tag}_ref_nit_nfev"][:, 1]
        print(tag, "records", out[f"{tag}_ref_dets"].shape[0], "nfev max", int(nf.max()), "at cap", int((nf == 200).sum()))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "det_post.npz"), **out)


if __name__ == "__main__":
    main()
