"""float64 / scipy restatement of the reference's scorer, the oracle of posecnn_b200/evaluate.py (DESIGN.md §14).

    fast_hist          lib/datasets/imdb.py:123-125
    quat2mat           transforms3d.quaternions.quat2mat (what lov.py:587 calls), on float64
    re / te / add / adi / reproj   lib/utils/pose_error.py (numpy, scipy.spatial.cKDTree), with the reference's dtypes: the estimate's
                       RT is float32 (lov.py:586-588), the gt pose float64 (scipy.io.loadmat of the dataset's meta .mat)
    score              the pairing loops of lov.py:576-628 with the eggbox rule and the 5-pixel count of linemod.py:700-760
    summary            lov.py:645-680
make_case builds the seeded inputs of tests/golden/eval.npz (tests/golden/make_golden_eval.py runs the reference's own
pose_error.py on them)."""
from __future__ import annotations

import math

import numpy as np
from scipy import spatial

from posecnn_b200 import synth

FLOAT_EPS = np.finfo(np.float64).eps          # transforms3d.quaternions._FLOAT_EPS


def fast_hist(a, b, n):
    k = (a >= 0) & (a < n)                                                                   # imdb.py:124
    return np.bincount(n * a[k].astype(int) + b[k].astype(int), minlength=n ** 2).reshape(n, n)   # imdb.py:125


def quat2mat(q):
    """transforms3d.quaternions.quat2mat on the float64 values of q = (w, x, y, z)."""
    w, x, y, z = (float(v) for v in q)
    Nq = w * w + x * x + y * y + z * z
    if Nq < FLOAT_EPS:
        return np.eye(3)
    s = 2.0 / Nq
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                     [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def transform_pts_Rt(pts, R, t):                                  # pose_error.py:12-22
    return (R.dot(pts.T) + t.reshape((3, 1))).T


def re(R_est, R_gt):                                              # pose_error.py:93-107
    error_cos = 0.5 * (np.trace(R_est.dot(np.linalg.inv(R_gt))) - 1.0)
    error_cos = min(1.0, max(-1.0, error_cos))
    return 180.0 * math.acos(error_cos) / np.pi


def te(t_est, t_gt):                                              # pose_error.py:109-119
    return np.linalg.norm(t_gt - t_est)


def add(R_est, t_est, R_gt, t_gt, pts):                          # pose_error.py:54-68
    return np.linalg.norm(transform_pts_Rt(pts, R_est, t_est) - transform_pts_Rt(pts, R_gt, t_gt), axis=1).mean()


def adi(R_est, t_est, R_gt, t_gt, pts):                          # pose_error.py:70-91
    nn_dists, _ = spatial.cKDTree(transform_pts_Rt(pts, R_est, t_est)).query(transform_pts_Rt(pts, R_gt, t_gt), k=1)
    return nn_dists.mean()


def reproj(K, R_est, t_est, R_gt, t_gt, pts):                    # pose_error.py:24-52
    def pix(P):
        p = K.dot(P.T).T
        out = np.zeros((P.shape[0], 2), dtype=np.float32)
        out[:, 0] = p[:, 0] / p[:, 2]
        out[:, 1] = p[:, 1] / p[:, 2]
        return out
    return np.linalg.norm(pix(transform_pts_Rt(pts, R_est, t_est)) - pix(transform_pts_Rt(pts, R_gt, t_gt)), axis=1).mean()


def se3_mul(RT1, RT2):                                           # utils/se3.py:19-30
    RT_new = np.zeros((3, 4), dtype=np.float32)
    RT_new[0:3, 0:3] = np.dot(RT1[0:3, 0:3], RT2[0:3, 0:3])
    RT_new[0:3, 3] = (np.dot(RT1[0:3, 0:3], RT2[0:3, 3].reshape((3, 1))) + RT1[0:3, 3].reshape((3, 1))).reshape((3))
    return RT_new


def estimate_rt(pose7):
    """lov.py:586-588: RT = float32 [quat2mat(q) | t]."""
    RT = np.zeros((3, 4), dtype=np.float32)
    RT[:3, :3] = quat2mat(pose7[:4])
    RT[:, 3] = pose7[4:7]
    return RT


def score(gt_rows, rois, pose_sets, num_rows, meta, points, symmetric, threshold, flip_z, C, batch_offset=0, fns=None):
    """The loops of lov.py:576-628 / linemod.py:700-760 over one batch.  gt_rows [n,14] f32, rois [cap,>=2], pose_sets: list of
    [cap,7], num_rows: rows scored, meta [B,>=9] (K = meta[b, :9]).  fns: the pose_error functions and se3_mul (default: this module's).
    Returns pairs [n_pairs,2] int32 (gt, row), errors [S,n_pairs,4] f64, flags [S,n_pairs] int32, counts [S,3,C] int64."""
    f = fns or dict(re=re, te=te, add=add, adi=adi, reproj=reproj, se3_mul=se3_mul)
    S = len(pose_sets)
    counts = np.zeros((S, 3, C), np.int64)
    pairs, errors, flags = [], [[] for _ in range(S)], [[] for _ in range(S)]
    for j in range(gt_rows.shape[0]):
        b, cls = int(gt_rows[j, 0]), int(gt_rows[j, 1])
        if not 0 < cls < C:                                      # lov.py:577-578
            continue
        counts[:, 0, cls] += 1                                   # lov.py:580
        R_gt = gt_rows[j, 2:].reshape(3, 4)[:, :3].astype(np.float64)
        t_gt = gt_rows[j, 2:].reshape(3, 4)[:, 3].astype(np.float64)
        K = meta[b - batch_offset, :9].astype(np.float64).reshape(3, 3)
        pts = points[cls]
        for k in range(num_rows):                                # lov.py:582-584
            if int(rois[k, 0]) != b or int(rois[k, 1]) != cls:
                continue
            pairs.append((j, k))
            for s in range(S):
                RT = estimate_rt(pose_sets[s][k])
                e_r = f["re"](RT[:3, :3], R_gt)                  # lov.py:599-600
                e_t = f["te"](RT[:, 3], t_gt)
                flip = flip_z[cls] > 0 and e_r > 90              # linemod.py:727-733
                if flip:
                    RT_z = np.array([[-1, 0, 0, 0], [0, -1, 0, 0], [0, 0, 1, 0]])
                    RT_sym = f["se3_mul"](RT, RT_z)
                    e_px = f["reproj"](K, RT_sym[:3, :3], RT_sym[:, 3], R_gt, t_gt, pts)
                else:
                    e_px = f["reproj"](K, RT[:3, :3], RT[:, 3], R_gt, t_gt, pts)
                dist = f["adi"] if symmetric[cls] > 0 else f["add"]   # lov.py:601-604
                e = dist(RT[:3, :3], RT[:, 3], R_gt, t_gt, pts)
                ok, ok_px = e < threshold[cls], e_px < 5         # lov.py:606, linemod.py:732
                counts[s, 1, cls] += ok
                counts[s, 2, cls] += ok_px
                errors[s].append((e_r, e_t, e, e_px))
                flags[s].append(int(ok) | 2 * int(ok_px) | 4 * int(flip))
    return (np.array(pairs, np.int32).reshape(-1, 2), np.array(errors, np.float64).reshape(S, -1, 4),
            np.array(flags, np.int32).reshape(S, -1), counts)


def summary(hist, counts, set_names):
    """lov.py:645-680 (accuracy NaN where count_all is 0)."""
    hist = hist.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        acc_cls = np.diag(hist) / hist.sum(1)
        iu = np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))
        freq = hist.sum(1) / hist.sum()
        out = dict(overall_accuracy=np.diag(hist).sum() / hist.sum(), mean_accuracy=np.nanmean(acc_cls), per_class_iu=iu,
                   mean_iu=np.nanmean(iu), fwavacc=(freq[freq > 0] * iu[freq > 0]).sum(), poses={})
        for s, name in enumerate(set_names):
            a, c, p = counts[s].astype(np.int64)
            out["poses"][name] = dict(count_all=a, count_correct=c, count_pixel=p, accuracy=c / a, accuracy_pixel=p / a)
    return out


def default_threshold(extents):
    """lov.py:539-541: threshold[i] = 0.1 * ||extents[i]||, stored in a float32 array."""
    return np.array([0.1 * np.linalg.norm(e) for e in np.asarray(extents, np.float32)], np.float32)


def _rot(axis, deg):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    h = 0.5 * np.deg2rad(deg)
    return np.r_[np.cos(h), np.sin(h) * axis]


def _qmul(a, b):
    w0, v0, w1, v1 = a[0], a[1:], b[0], b[1:]
    return np.r_[w0 * w1 - v0 @ v1, w0 * v1 + w1 * v0 + np.cross(v0, v1)]


def make_case(tag):
    """Seeded inputs of one golden case.  "lov": C = 22, two 48x64 images with gt = -1 pixels, five objects per image (the
    symmetric classes 13, 16, 21 among them), a gt with no detection, a background gt row, duplicate detections, three pose sets
    (near-identity errors down to 1e-4 degrees, a zero quaternion, large errors), 7-column rois.  "egg": C = 2 with the eggbox
    flip and ADD-S on class 1, estimates on both sides of 90 degrees, 6-column rois, num_rows < cap."""
    rng = np.random.default_rng({"lov": 101, "egg": 202}[tag])
    C, B, H, W = (22, 2, 48, 64) if tag == "lov" else (2, 2, 40, 56)
    K = synth.intrinsics(480, 640)
    meta = np.stack([synth.make_meta(K)] * B).astype(np.float32)
    gt_label = rng.integers(0, C, (B, H, W)).astype(np.int32)
    gt_label[:, :8] = 0
    gt_label[:, -4:] = -1
    label = np.where(rng.random((B, H, W)) < 0.7, np.maximum(gt_label, 0), rng.integers(0, C, (B, H, W))).astype(np.int32)
    if tag == "lov":
        classes = [[13, 16, 5, 21, 2], [1, 13, 7, 9, 21]]
    else:
        classes = [[1], [1, 1]]
    gt_rows, rows, sets = [], [], [[], [], []]
    angles = [1e-4, 1e-3, 0.05, 2.0, 20.0] if tag == "lov" else [30.0, 89.0, 91.0, 150.0, 179.0]
    for b in range(B):
        for i, cls in enumerate(classes[b]):
            q = synth._rand_quat(rng)
            t = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.15, 0.15), rng.uniform(0.6, 1.2)])
            RT = np.zeros((3, 4), np.float32)
            RT[:, :3] = quat2mat(q)
            RT[:, 3] = t
            gt_rows.append(np.r_[b, cls, RT.reshape(-1)])
            if tag == "lov" and b == 1 and i == 4:
                continue                                         # a gt without a detection
            ndet = 2 if i == 1 else 1                            # duplicate detections of one class
            for d in range(ndet):
                rows.append([b, cls])
                for s in range(3):
                    ang = angles[(i + d + s) % len(angles)]
                    qe = _qmul(_rot(rng.normal(size=3), ang), q)
                    te_ = t + rng.normal(0, 1e-3 * (s + 1), 3)
                    if tag == "lov" and b == 0 and i == 2 and s == 1:
                        qe = np.zeros(4)                         # a zero quaternion: quat2mat's identity branch
                    if s == 2 and d == 1:
                        qe, te_ = q * 1.0, t.copy()              # the gt pose itself (acos at 1)
                    sets[s].append(np.r_[qe, te_])
    if tag == "lov":
        gt_rows.append(np.r_[0, 0, np.eye(3, 4).reshape(-1)])     # class 0: skipped
        rows.append([1, 3])                                      # a detection of a class without gt
        for s in range(3):
            sets[s].append(np.r_[1.0, 0, 0, 0, 0, 0, 1.0])
    n = len(rows)
    cap = n + 3
    ncol = 7 if tag == "lov" else 6
    rois = np.zeros((cap, ncol), np.float32)
    rois[:n, :2] = rows
    rois[:n, 2:] = rng.uniform(0, 100, (n, ncol - 2))
    rois[n:, 1] = rois[:n, 1][: cap - n]                         # rows past num_rows that would pair: must be ignored
    poses = np.zeros((3, cap, 7), np.float32)
    poses[:, :n] = np.array(sets, np.float32)
    poses[:, n:] = poses[:, :cap - n]
    num_rows = n if tag == "lov" else n - 1
    ext = synth.extents_for(C)
    symmetric = np.zeros(C, np.float32)
    flip_z = np.zeros(C, np.float32)
    if tag == "lov":
        symmetric[[13, 16, 21]] = 1
    else:
        symmetric[1] = 1
        flip_z[1] = 1
    return dict(C=C, gt_label=gt_label, label=label, gt_rows=np.array(gt_rows, np.float32), rois=rois, poses=poses,
                num_rows=num_rows, meta=meta, extents=ext, symmetric=symmetric, flip_z=flip_z, threshold=default_threshold(ext))


CASES = ("lov", "egg")
