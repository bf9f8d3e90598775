"""ctypes front-end of the CPU oracle (oracle/posecnn_oracle.c).

TEST INFRASTRUCTURE ONLY — importable from tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py.  The product package
(posecnn_b200/) never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
MAX_ROWS = 128 * 9


def build(force: bool = False) -> str:
    """Compile the C restatement with gcc (seconds)."""
    so = os.path.join(_HERE, "_build", "libposecnn_oracle.so")
    src = os.path.join(_HERE, "posecnn_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "_build/libposecnn_oracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
    return _LIB


def _p(a, t=ctypes.c_float):
    if a is None:
        return None
    return a.ctypes.data_as(ctypes.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def hough_voting_gpu(label, vertex, extents, meta, gt, is_train=0, threshold_vote=-1.0, threshold_percentage=0.02,
                     skip_pixels=10, inlier_threshold=0.9, label_threshold=500, debug=False, slack=False):
    """Canonical-order restatement of Houghvotinggpu.  Returns the five op outputs
    (with the >=1 dummy-row rule of hough_voting_gpu_op.cc:379-383) and, if debug,
    a dict with the raw row count, vote planes and ambiguity counts; with slack=True (implies debug) also the
    exactness analysis of the interval scan: `slack` [B,C,H,W] int32 (irregular (sample, row) pairs whose window row
    holds the cell) and `pairs` [B,C,2] int64 ((sample, row) pairs inside a window, irregular ones)."""
    debug = debug or slack
    label = _i32(label); vertex = _f32(vertex); extents = _f32(extents); meta = _f32(meta)
    gt = np.zeros((0, 13), np.float32) if gt is None else _f32(gt).reshape(-1, 13)
    B, H, W = label.shape
    C = vertex.shape[3] // 3
    num_meta = meta.shape[-1]
    box = np.zeros((MAX_ROWS, 7), np.float32); pose = np.zeros((MAX_ROWS, 7), np.float32)
    target = np.zeros((MAX_ROWS, 4 * C), np.float32); weight = np.zeros((MAX_ROWS, 4 * C), np.float32)
    domain = np.zeros((MAX_ROWS,), np.int32)
    nrois = ctypes.c_int(0)
    votes = np.zeros((B, C, H, W), np.float32) if debug else None
    ambig = np.zeros((B, C, H, W), np.int32) if debug else None
    slk = np.zeros((B, C, H, W), np.int32) if slack else None
    pairs = np.zeros((B, C, 2), np.int64) if slack else None
    gt_arg = gt if gt.size else np.zeros((1, 13), np.float32)
    rc = lib().pcnn_oracle_hough(
        _p(label, ctypes.c_int), _p(vertex), _p(extents), _p(meta), _p(gt_arg), B, H, W, C, gt.shape[0], num_meta,
        int(is_train), ctypes.c_float(inlier_threshold), int(label_threshold), ctypes.c_float(threshold_vote),
        ctypes.c_float(threshold_percentage), int(skip_pixels), _p(box), _p(pose), _p(target), _p(weight),
        _p(domain, ctypes.c_int), ctypes.byref(nrois), _p(votes), _p(ambig, ctypes.c_int), _p(slk, ctypes.c_int),
        _p(pairs, ctypes.c_longlong))
    assert rc == 0
    n = max(1, nrois.value)
    outs = (box[:n].copy(), pose[:n].copy(), target[:n].copy(), weight[:n].copy(), domain[:n].copy())
    if debug:
        dbg = dict(num_rois=nrois.value, votes=votes, ambig=ambig)
        if slack:
            dbg.update(slack=slk, pairs=pairs)
        return outs, dbg
    return outs


def project_box(extents, meta, cls, distance, factor=0.6):
    """project_box (.cu.cc:84-120) of one image's meta record: the half-size of a sample's vote window at depth distance."""
    f = lib().pcnn_oracle_project_box
    f.restype = ctypes.c_float
    return f(int(cls), _p(_f32(extents)), _p(_f32(meta).reshape(-1)), ctypes.c_float(distance), ctypes.c_float(factor))


def hough_row_exact(passes, wmin, x, own_row):
    """The exactness criterion of one (sample, row) pair (pcnn_oracle_hough_row_exact): `passes` = the reference
    predicate on the window row's cells wmin .. wmin + len - 1; True when the set is empty or one interval (on the
    pixel's own row: empty or one whole side of the window)."""
    p = np.ascontiguousarray(passes, dtype=np.uint8)
    return bool(lib().pcnn_oracle_hough_row_exact(_p(p, ctypes.c_ubyte), int(wmin), int(wmin) + p.size - 1, int(x),
                                                  int(bool(own_row))))


def roi_pool(data, rois, pooled_height, pooled_width, spatial_scale, pool_channel=0):
    data = _f32(data); rois = _f32(rois)
    B, H, W, Cc = data.shape
    N, cr = rois.shape
    co = 1 if pool_channel else Cc
    top = np.zeros((N, pooled_height, pooled_width, co), np.float32)
    arg = np.zeros((N, pooled_height, pooled_width, co), np.int32)
    lib().pcnn_oracle_roi_pool_fwd(_p(data), _p(rois), N, cr, H, W, Cc, pooled_height, pooled_width,
                                   ctypes.c_float(spatial_scale), int(pool_channel), _p(top), _p(arg, ctypes.c_int))
    return top, arg


def roi_pool_grad(data, rois, argmax, grad, pooled_height, pooled_width, spatial_scale, pool_channel=0):
    data = _f32(data); rois = _f32(rois); argmax = _i32(argmax); grad = _f32(grad)
    B, H, W, Cc = data.shape
    N, cr = rois.shape
    out = np.zeros_like(data)
    lib().pcnn_oracle_roi_pool_bwd(_p(grad), _p(argmax, ctypes.c_int), _p(rois), B, N, cr, H, W, Cc, pooled_height,
                                   pooled_width, ctypes.c_float(spatial_scale), int(pool_channel), _p(out))
    return out


def hard_label(prob, gt, threshold):
    prob = _f32(prob); gt = _i32(gt)
    C = prob.shape[-1]
    top = np.empty_like(prob)
    lib().pcnn_oracle_hard_label(_p(prob), _p(gt, ctypes.c_int), ctypes.c_long(gt.size), C,
                                 ctypes.c_float(threshold), _p(top))
    return top


def project(data, depth, meta, kernel_size=0, threshold=0.0, return_ambig=False):
    """ProjectForward: data [B,G,G,G,Cf] -> [B,H,W,Cf]."""
    data = _f32(data); depth = _f32(depth); meta = _f32(meta)
    B, G = data.shape[0], data.shape[1]
    Cf = data.shape[4]
    H, W = depth.shape[1], depth.shape[2]
    out = np.zeros((B, H, W, Cf), np.float32)
    amb = np.zeros((B, H, W), np.uint8)
    lib().pcnn_oracle_pixel_gather(_p(data), _p(depth), _p(meta), B, H, W, Cf, meta.shape[-1], G, _p(out),
                                   _p(amb, ctypes.c_ubyte))
    return (out, amb.astype(bool)) if return_ambig else out


def backproject_grad(top_diff, depth, meta, return_ambig=False):
    """BackprojectBackward has ProjectForward's gather semantics on top_diff."""
    return project(top_diff, depth, meta, return_ambig=return_ambig)


def backproject(data, label, depth, meta, label_3d, grid_size, kernel_size, threshold, return_ambig=False):
    data = _f32(data); label = _f32(label); depth = _f32(depth); meta = _f32(meta); label_3d = _f32(label_3d)
    B, H, W, Cf = data.shape
    C = label.shape[3]
    G = grid_size
    td = np.zeros((B, G, G, G, Cf), np.float32); tl = np.zeros((B, G, G, G, C), np.float32)
    tf = np.zeros((B, G, G, G, Cf), np.float32); amb = np.zeros((B, G, G, G), np.uint8)
    lib().pcnn_oracle_voxel_average(_p(data), _p(label), _p(depth), _p(meta), _p(label_3d), B, H, W, Cf, C,
                                    meta.shape[-1], G, int(kernel_size), ctypes.c_float(threshold), _p(td), _p(tl),
                                    _p(tf), _p(amb, ctypes.c_ubyte))
    return (td, tl, tf, amb.astype(bool)) if return_ambig else (td, tl, tf)


def project_grad(top_diff, depth, meta, grid_size, kernel_size, threshold, return_ambig=False):
    """ProjectBackward: window average of top_diff [B,H,W,Cf] into [B,G,G,G,Cf]."""
    top_diff = _f32(top_diff); depth = _f32(depth); meta = _f32(meta)
    B, H, W, Cf = top_diff.shape
    G = grid_size
    out = np.zeros((B, G, G, G, Cf), np.float32); amb = np.zeros((B, G, G, G), np.uint8)
    lib().pcnn_oracle_voxel_average(_p(top_diff), None, _p(depth), _p(meta), None, B, H, W, Cf, 0, meta.shape[-1], G,
                                    int(kernel_size), ctypes.c_float(threshold), _p(out), None, None,
                                    _p(amb, ctypes.c_ubyte))
    return (out, amb.astype(bool)) if return_ambig else out


def voxel_window(depth, meta, grid_size, kernel_size, threshold):
    """The windows of Backproject / ProjectGrad: per voxel [B,G,G,G] the hit count (int32) and whether the image border
    clips the window (bool)."""
    depth = _f32(depth); meta = _f32(meta)
    B, H, W = depth.shape[0], depth.shape[1], depth.shape[2]
    G = grid_size
    count = np.zeros((B, G, G, G), np.int32); clipped = np.zeros((B, G, G, G), np.uint8)
    lib().pcnn_oracle_voxel_window(_p(depth), _p(meta), B, H, W, meta.shape[-1], G, int(kernel_size),
                                   ctypes.c_float(threshold), _p(count, ctypes.c_int), _p(clipped, ctypes.c_ubyte))
    return count, clipped.astype(bool)


def average_distance_loss(pred, target, weight, point, symmetry, margin):
    pred = _f32(pred); target = _f32(target); weight = _f32(weight); point = _f32(point); symmetry = _f32(symmetry)
    N = pred.shape[0]
    C, P = point.shape[0], point.shape[1]
    loss = ctypes.c_float(0)
    diff = np.zeros((N, 4 * C), np.float32)
    near = ctypes.c_int(0)
    lib().pcnn_oracle_average_distance(_p(pred), _p(target), _p(weight), _p(point), _p(symmetry), N, C, P,
                                       ctypes.c_float(margin), ctypes.byref(loss), _p(diff), ctypes.byref(near))
    return np.array([loss.value], np.float32), diff


# ---------------------------------------------------------------------------------------------------------------
# Test-time post-processing (SURVEY.md §8(f) rank 1), numpy restatement
# ---------------------------------------------------------------------------------------------------------------
def nms(dets, thresh, per_image=False):
    """lib/utils/nms.py:3-32 restated: greedy NMS in descending score order over rows
    [batch, cls, x1, y1, x2, y2, score]; a later box is dropped when IoU(+1 convention) > thresh with a kept box of the
    same class.  float32 arithmetic as numpy does on float32 rows.  Canonical tie order: stable ascending argsort,
    reversed (the reference's default-kind argsort()[::-1] is not stable for n > 16).  per_image=True additionally
    requires the same batch index (the reference ignores the batch column; it only ever runs batch 1)."""
    dets = np.asarray(dets, dtype=np.float32)
    if dets.shape[0] == 0:
        return []
    cls, x1, y1, x2, y2, scores = (dets[:, k] for k in (1, 2, 3, 4, 5, 6))
    img = dets[:, 0].astype(np.int64)
    areas = (x2 - x1 + np.float32(1)) * (y2 - y1 + np.float32(1))        # nms.py:12
    order = scores.argsort(kind="stable")[::-1]                           # nms.py:13 (canonical tie order)
    keep = []
    while order.size > 0:                                                 # nms.py:16-30
        i = order[0]
        keep.append(int(i))
        rest = order[1:]
        xx1 = np.maximum(x1[i], x1[rest]); yy1 = np.maximum(y1[i], y1[rest])
        xx2 = np.minimum(x2[i], x2[rest]); yy2 = np.minimum(y2[i], y2[rest])
        w = np.maximum(np.float32(0), xx2 - xx1 + np.float32(1))
        h = np.maximum(np.float32(0), yy2 - yy1 + np.float32(1))
        inter = w * h
        ovr = inter / (areas[i] + areas[rest] - inter)
        same = cls[rest] == cls[i]
        if per_image:
            same &= img[rest] == img[i]
        order = rest[~((ovr > np.float32(thresh)) & same)]
    if per_image:   # images are independent: emit them in batch order (processing order inside an image), like the op's batch loop
        keep = sorted(keep, key=lambda k: int(img[k]))      # stable: keeps the processing order inside an image
    return keep


def assemble_poses(rois, poses_init, poses_pred, keep):
    """lib/fcn/test.py:197-211: rows [keep]; poses[i, :4] = poses_pred[i, 4c:4c+4] for class c = rois[i, 1] >= 0."""
    rois = np.asarray(rois, np.float32)[keep]
    poses = np.array(np.asarray(poses_init, np.float32)[keep], copy=True)
    if poses_pred is not None:
        pp = np.asarray(poses_pred, np.float32)[keep]
        for i in range(rois.shape[0]):
            c = int(rois[i, 1])
            if c >= 0:
                poses[i, :4] = pp[i, 4 * c:4 * c + 4]
    return rois, poses


# ---------------------------------------------------------------------------------------------------------------
# Training-side targets and losses (SURVEY.md §8(f) rank 3), numpy restatements
# ---------------------------------------------------------------------------------------------------------------
def generate_vertex_targets(label, centers, w_inside):
    """lib/gt_synthesize_layer/minibatch.py:578-599 (single-instance branch, VERTEX_REG_2D): label [B,H,W] int32,
    centers [B,C,3] = (cx, cy, z), z <= 0 = class not in cls_indexes.  float32 centre - int64 pixel grid = float64
    arithmetic, stored into float32 arrays."""
    label = np.asarray(label)
    B, H, W = label.shape
    C = centers.shape[1]
    targets = np.zeros((B, H, W, 3 * C), np.float32)
    weights = np.zeros((B, H, W, 3 * C), np.float32)
    for b in range(B):
        for i in range(1, C):                                             # :579
            y, x = np.where(label[b] == i)                                # :580
            if len(x) > 0 and centers[b, i, 2] > 0:                       # :583 (class listed in cls_indexes)
                c = np.zeros((2, 1), np.float32)
                c[0], c[1] = centers[b, i, 0], centers[b, i, 1]           # :585-586
                z = centers[b, i, 2]
                R = np.tile(c, (1, len(x))) - np.vstack((x, y))           # :588  (float64)
                N = np.linalg.norm(R, axis=0) + 1e-10                     # :590
                R = np.divide(R, np.tile(N, (2, 1)))                      # :592
                targets[b, y, x, 3 * i + 0] = R[0, :]                     # :594-596
                targets[b, y, x, 3 * i + 1] = R[1, :]
                targets[b, y, x, 3 * i + 2] = np.log(np.float64(z))
                weights[b, y, x, 3 * i:3 * i + 3] = w_inside              # :600-602
    return targets, weights


def generate_vertex_targets_instances(label, mask, instances, num_classes, w_inside):
    """lib/gt_synthesize_layer/minibatch.py:549-573 (multi-instance branch, VERTEX_REG_2D): instances [B,I,5] =
    (cls, mask id = cls_indexes_old + 1, cx, cy, z), z <= 0 = unused slot; in-order overwrites like the reference loop."""
    label, mask = np.asarray(label), np.asarray(mask)
    B, H, W = label.shape
    C = num_classes
    targets = np.zeros((B, H, W, 3 * C), np.float32)
    weights = np.zeros((B, H, W, 3 * C), np.float32)
    for b in range(B):
        for r in instances[b]:
            if not r[4] > 0:
                continue
            cls = int(r[0])
            y, x = np.where((mask[b] == int(r[1])) & (label[b] == cls))   # :553
            if len(x) > 0:
                c = np.zeros((2, 1), np.float32)
                c[0], c[1] = r[2], r[3]                                   # :557-558
                R = np.tile(c, (1, len(x))) - np.vstack((x, y))           # :560
                N = np.linalg.norm(R, axis=0) + 1e-10
                R = np.divide(R, np.tile(N, (2, 1)))
                targets[b, y, x, 3 * cls + 0] = R[0, :]
                targets[b, y, x, 3 * cls + 1] = R[1, :]
                targets[b, y, x, 3 * cls + 2] = np.log(np.float64(r[4]))
                weights[b, y, x, 3 * cls:3 * cls + 3] = w_inside
    return targets, weights


def mat2quat(M):
    """transforms3d.quaternions.mat2quat (third-party, un-pinned, absent here: `from transforms3d.quaternions import
    mat2quat`, minibatch.py:18) restated from its published algorithm (Bar-Itzhack 2000): the eigenvector of the largest
    eigenvalue of the symmetric K matrix, ordered (w, x, y, z), w made non-negative.  Parity unpinned for this function;
    cross-checked against scipy.spatial.transform.Rotation in tests/test_golden_cpu.py."""
    Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = np.asarray(M, np.float64).flat
    K = np.array([[Qxx - Qyy - Qzz, 0, 0, 0],
                  [Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0],
                  [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0],
                  [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3.0
    vals, vecs = np.linalg.eigh(K)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    if q[0] < 0:
        q = -q
    return q


def pack_pose_meta(poses, cls, intrinsics, im_scale=1.0, flip_x=False):
    """minibatch.py:440-451 (pose blob rows [image, cls, 0,0,0,0, mat2quat(R), T]) and :474-492 (meta_data[48]):
    poses [B,I,3,4], cls [B,I] (< 0 = unused slot), intrinsics [B,3,3]."""
    B, I = cls.shape
    rows = []
    for b in range(B):
        for j in range(I):
            if cls[b, j] < 0:
                continue
            qt = np.zeros(13, np.float32)
            qt[0], qt[1] = b, cls[b, j]
            qt[6:10] = mat2quat(poses[b, j, :, :3])
            qt[10:] = poses[b, j, :, 3]
            rows.append(qt)
    blob = np.stack(rows) if rows else np.zeros((0, 13), np.float32)
    meta = np.zeros((B, 48), np.float32)
    for b in range(B):
        K = np.asarray(intrinsics[b], np.float32).astype(np.float64) * im_scale
        K[2, 2] = 1
        meta[b, 0:9] = K.flatten()
        meta[b, 9:18] = np.linalg.pinv(K).flatten()
        if flip_x:
            meta[b, 0] = -meta[b, 0]; meta[b, 9] = -meta[b, 9]; meta[b, 11] = -meta[b, 11]
    return blob, meta


def loss_cross_entropy_hard(scores, prob, gt, threshold):
    """lib/fcn/train.py:455-465 with labels = Hardlabel(prob, gt, threshold) (network.py:340): float64 accumulation."""
    mask = hard_label(np.asarray(prob, np.float32), np.asarray(gt, np.int32), threshold).astype(np.float64)
    ce = -(mask * np.asarray(scores, np.float64)).sum(axis=3)
    return ce.sum() / (mask.sum() + 1e-10), mask


def smooth_l1_loss_vertex(pred, targets, weights, sigma=1.0):
    """lib/fcn/train.py:564-573 in float32 element arithmetic, float64 accumulation.  Returns (loss, d loss / d pred)."""
    s2 = np.float32(sigma) ** 2
    diff = np.asarray(weights, np.float32) * (np.asarray(pred, np.float32) - np.asarray(targets, np.float32))
    ad = np.abs(diff)
    sign = (ad < np.float32(1.0) / s2).astype(np.float32)
    in_loss = diff * diff * (s2 / np.float32(2)) * sign + (ad - np.float32(0.5) / s2) * (np.float32(1) - sign)
    wsum = np.asarray(weights, np.float64).sum() + 1e-10
    g = np.where(sign > 0, diff * s2, np.sign(diff)) * np.asarray(weights, np.float32)
    return in_loss.astype(np.float64).sum() / wsum, (g / wsum).astype(np.float32)
