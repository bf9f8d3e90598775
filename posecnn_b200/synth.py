"""Deterministic synthetic inputs for the PoseCNN hot path (SURVEY.md §8(d)).

The reference ships no test fixtures (SURVEY.md §4), and its datasets cannot be
fetched here, so every parity test and benchmark runs on scenes produced by this
generator.  Shapes, layouts and value conventions follow the reference's data
layer:

* label / vertex target layout ........ lib/gt_synthesize_layer/minibatch.py:543-602
  (per class c, channels 3c..3c+2 = unit direction to the object centre, log z)
* meta_data[48] packing ................ lib/fcn/test.py:121-149
* gt pose rows [b, cls, 0,0,0,0, qw,qx,qy,qz, tx,ty,tz] .. minibatch.py:440-451
* camera intrinsics .................... tools/demo.py:100-101
* object extents ....................... data/LOV/extents.txt (values restated below;
  row 0 = background = 0, lib/datasets/lov.py:161-170)
* symmetry flags ....................... lib/datasets/lov.py:38

Everything is numpy; nothing here touches the GPU or the oracle.
"""
from __future__ import annotations

import numpy as np

# data/LOV/extents.txt — physical extents (metres) of the 21 YCB-Video objects.
LOV_EXTENTS = np.array(
    [
        [0.0, 0.0, 0.0],
        [0.105098, 0.103336, 0.147140],
        [0.072948, 0.167432, 0.223122],
        [0.051228, 0.097062, 0.184740],
        [0.068346, 0.070898, 0.118506],
        [0.099712, 0.071530, 0.215002],
        [0.085656, 0.085848, 0.041788],
        [0.140458, 0.136312, 0.044982],
        [0.092226, 0.102030, 0.037278],
        [0.106770, 0.061462, 0.099400],
        [0.146328, 0.202874, 0.039542],
        [0.159810, 0.157306, 0.293620],
        [0.112422, 0.072590, 0.277178],
        [0.161696, 0.163252, 0.060978],
        [0.133400, 0.094318, 0.084588],
        [0.202122, 0.229442, 0.061552],
        [0.106668, 0.108480, 0.240242],
        [0.110210, 0.257878, 0.015808],
        [0.021110, 0.125212, 0.019532],
        [0.140818, 0.174792, 0.040068],
        [0.210450, 0.185262, 0.036514],
        [0.052900, 0.077960, 0.067918],
    ],
    dtype=np.float32,
)

# lib/datasets/lov.py:38
LOV_SYMMETRY = np.array(
    [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1], dtype=np.float32
)

# tools/demo.py:100-101 / data/LOV/camera.json:14
FX, FY, PX, PY = 1066.778, 1067.487, 312.9869, 241.3109
PIXEL_MEANS = np.array([102.9801, 115.9465, 122.7717], dtype=np.float32)  # lib/fcn/config.py:242


def extents_for(num_classes: int) -> np.ndarray:
    """[C,3] extents; C<=22 takes the first C rows, larger C cycles the objects."""
    if num_classes <= LOV_EXTENTS.shape[0]:
        return LOV_EXTENTS[:num_classes].copy()
    rows = [LOV_EXTENTS[0]]
    for c in range(1, num_classes):
        rows.append(LOV_EXTENTS[1 + (c - 1) % 21])
    return np.stack(rows).astype(np.float32)


def intrinsics(height: int = 480, width: int = 640) -> np.ndarray:
    """3x3 K scaled from the 640x480 YCB camera to (height, width)."""
    sx, sy = width / 640.0, height / 480.0
    return np.array([[FX * sx, 0, PX * sx], [0, FY * sy, PY * sy], [0, 0, 1]], dtype=np.float64)


def make_meta(K: np.ndarray, grid_size: int = 128, rt_w2l: np.ndarray | None = None) -> np.ndarray:
    """48-float meta_data record (lib/fcn/test.py:121-149)."""
    m = np.zeros(48, dtype=np.float32)
    m[0:9] = K.reshape(-1)
    m[9:18] = np.linalg.pinv(K).reshape(-1)
    if rt_w2l is None:
        rt_w2l = np.hstack([np.eye(3), np.zeros((3, 1))])
    T = np.vstack([rt_w2l, [0, 0, 0, 1]])
    m[18:30] = rt_w2l.reshape(-1)
    m[30:42] = np.linalg.inv(T)[:3].reshape(-1)
    m[42:45] = (6.0 / grid_size, 6.0 / grid_size, 7.0 / grid_size)
    m[45:48] = (-3.0, -3.0, -3.0)
    return m


def _rand_quat(rng) -> np.ndarray:
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    if q[0] < 0:
        q = -q
    return q


def make_scene(
    batch: int = 1,
    height: int = 480,
    width: int = 640,
    num_classes: int = 22,
    objects_per_image: int | None = None,
    seed: int = 1234,
    dir_noise: float = 0.05,
    min_pixels: int = 800,
    other_channel_noise: bool = True,
):
    """Synthetic label / vertex / meta / gt-pose tensors for the Hough path.

    Returns a dict of numpy arrays:
      label   [B,H,W]    int32
      vertex  [B,H,W,3C] float32
      extents [C,3]      float32
      meta    [B,1,1,48] float32
      gt      [num_gt,13] float32
      centers list of (b, cls, cx, cy, z) planted objects (after occlusion filtering)
    """
    C = num_classes
    if objects_per_image is None:
        objects_per_image = 5 if C >= 7 else 1
    K = intrinsics(height, width)
    fx, fy, px, py = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    ext = extents_for(C)
    label = np.zeros((batch, height, width), dtype=np.int32)
    vertex = np.empty((batch, height, width, 3 * C), dtype=np.float32)
    meta = np.zeros((batch, 1, 1, 48), dtype=np.float32)
    gt_rows = []
    centers = []
    ys, xs = np.mgrid[0:height, 0:width]
    for b in range(batch):
        rng = np.random.default_rng(seed + b)
        if other_channel_noise:
            vertex[b] = rng.standard_normal((height, width, 3 * C), dtype=np.float32)
        else:
            vertex[b] = 0
        meta[b, 0, 0] = make_meta(K)
        k = min(objects_per_image, C - 1)
        classes = rng.choice(np.arange(1, C), size=k, replace=False)
        placed = []
        for cls in classes:
            for _ in range(20):
                cx = rng.uniform(0.2 * width, 0.8 * width)
                cy = rng.uniform(0.2 * height, 0.8 * height)
                z = rng.uniform(0.6, 1.4)
                a = 0.5 * fx * ext[cls, 0] / z
                bb = 0.5 * fy * ext[cls, 1] / z
                mask = ((xs - cx) / a) ** 2 + ((ys - cy) / bb) ** 2 <= 1.0
                if mask.sum() >= min_pixels:
                    break
            else:
                continue
            label[b][mask] = cls
            placed.append((int(cls), cx, cy, z))
        for cls, cx, cy, z in placed:
            mask = label[b] == cls
            n = int(mask.sum())
            if n == 0:
                continue
            dx = cx - xs[mask]
            dy = cy - ys[mask]
            nrm = np.sqrt(dx * dx + dy * dy) + 1e-10
            u = dx / nrm + rng.normal(0, dir_noise, n)
            v = dy / nrm + rng.normal(0, dir_noise, n)
            vertex[b][mask, 3 * cls + 0] = u.astype(np.float32)
            vertex[b][mask, 3 * cls + 1] = v.astype(np.float32)
            vertex[b][mask, 3 * cls + 2] = np.float32(np.log(z))
            q = _rand_quat(rng)
            t = z * np.array([(cx - px) / fx, (cy - py) / fy, 1.0])
            gt_rows.append([b, cls, 0, 0, 0, 0, q[0], q[1], q[2], q[3], t[0], t[1], t[2]])
            centers.append((b, cls, cx, cy, z))
    gt = np.array(gt_rows, dtype=np.float32).reshape(-1, 13)
    return dict(label=label, vertex=vertex, extents=ext, meta=meta, gt=gt, centers=centers)


def make_model_points(num_classes: int = 22, num_points: int = 2620, seed: int = 7) -> np.ndarray:
    """[C,P,3] synthetic model point clouds: points on the ellipsoid inscribed in each
    class's extent box (the reference loads data/LOV/models/*/points.xyz,
    lib/datasets/lov.py:141-158, which cannot travel to the GPU box)."""
    rng = np.random.default_rng(seed)
    ext = extents_for(num_classes)
    pts = np.zeros((num_classes, num_points, 3), dtype=np.float32)
    for c in range(1, num_classes):
        d = rng.normal(size=(num_points, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        pts[c] = (d * ext[c] * 0.5).astype(np.float32)
    return pts


def quat_to_rot(q) -> np.ndarray:
    """(w, x, y, z) unit quaternion -> 3x3 rotation matrix."""
    w, x, y, z = (float(v) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def perturb_pose(q, t, rng, angle_deg: float = 3.0, lateral: float = 0.005, depth: float = 0.025):
    """A pose off by `angle_deg` about a random axis (applied in the camera frame), `lateral` metres in a random direction of the
    image plane and `depth` metres along z.  Returns (q [4], t [3]) float64."""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    h = 0.5 * np.deg2rad(angle_deg)
    dq = np.r_[np.cos(h), np.sin(h) * axis]
    w0, v0 = dq[0], dq[1:]
    w1, v1 = float(q[0]), np.asarray(q[1:], np.float64)
    qn = np.r_[w0 * w1 - v0 @ v1, w0 * v1 + w1 * v0 + np.cross(v0, v1)]
    phi = rng.uniform(0, 2 * np.pi)
    tn = np.asarray(t, np.float64) + np.array([lateral * np.cos(phi), lateral * np.sin(phi), depth])
    return qn, tn


def make_refine_scene(batch: int = 1, height: int = 480, width: int = 640, num_classes: int = 22, objects_per_image: int = 3,
                      seed: int = 5, noise_m: float = 0.0, factor_depth: float = 10000.0, num_points: int = 2620,
                      background_z: float = 1.8, min_pixels: int = 1500):
    """Depth scenes for the pose refiner: the ellipsoids of make_model_points (semi-axes extents / 2), posed, rendered
    analytically by ray-ellipsoid intersection with a z-buffer in front of a fronto-parallel background plane (label 0).

    Returns a dict of numpy arrays:
      label  [B,H,W] int32   class of the nearest surface
      depth  [B,H,W] f32     raw sensor units (metres * factor_depth), + N(0, noise_m) metres if noise_m > 0
      meta   [B,48]  f32     make_meta of the scaled YCB camera
      points [C,P,3] f32     make_model_points(num_classes, num_points)
      poses  [N,9]   f64     (b, cls, qw, qx, qy, qz, tx, ty, tz) of every object with >= min_pixels visible pixels
    """
    C = num_classes
    K = intrinsics(height, width)
    fx, fy, px, py = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    ext = extents_for(C)
    pts = make_model_points(C, num_points)
    vv, uu = np.mgrid[0:height, 0:width].astype(np.float64)
    rays = np.stack([(uu - px) / fx, (vv - py) / fy, np.ones_like(uu)], -1)
    label = np.zeros((batch, height, width), np.int32)
    depth = np.zeros((batch, height, width), np.float32)
    meta = np.zeros((batch, 48), np.float32)
    rows = []
    for b in range(batch):
        rng = np.random.default_rng(seed + 1000 * b)
        meta[b] = make_meta(K)
        zbuf = np.full((height, width), background_z)
        lab = np.zeros((height, width), np.int32)
        k = min(objects_per_image, C - 1)
        placed = []
        for cls in rng.choice(np.arange(1, C), size=k, replace=False):
            q = _rand_quat(rng)
            z = rng.uniform(0.6, 1.1)
            cx, cy = rng.uniform(0.25 * width, 0.75 * width), rng.uniform(0.25 * height, 0.75 * height)
            t = z * np.array([(cx - px) / fx, (cy - py) / fy, 1.0])
            R = quat_to_rot(q)
            inv_a = 1.0 / (0.5 * ext[cls].astype(np.float64))
            A = (rays @ R) * inv_a                     # R^T d, scaled
            Bv = -(R.T @ t) * inv_a
            aa = np.sum(A * A, -1)
            ab = A @ Bv
            disc = ab * ab - aa * (Bv @ Bv - 1.0)
            s = np.where(disc > 0, (-ab - np.sqrt(np.maximum(disc, 0))) / aa, np.inf)
            hit = (disc > 0) & (s > 0) & (s < zbuf)
            zbuf = np.where(hit, s, zbuf)
            lab[hit] = cls
            placed.append((int(cls), q, t))
        if noise_m > 0:
            zbuf = zbuf + rng.normal(0.0, noise_m, zbuf.shape)
        label[b] = lab
        depth[b] = (zbuf * factor_depth).astype(np.float32)
        for cls, q, t in placed:
            if int((lab == cls).sum()) >= min_pixels:
                rows.append([b, cls, *q, *t])
    return dict(label=label, depth=depth, meta=meta, points=pts, poses=np.array(rows, np.float64).reshape(-1, 9))


def make_coordinate_scene(batch: int = 1, height: int = 480, width: int = 640, num_classes: int = 22, objects_per_image: int = 3,
                          seed: int = 5, coord_noise_m: float = 0.0, outlier_fraction: float = 0.0, factor_depth: float = 10000.0):
    """Object-coordinate scenes for the VERTEX_REG_3D pose estimator, on the analytic ellipsoid scenes of make_refine_scene: the
    visible surface point X of a pixel is its ray scaled to the rendered depth, its object coordinate is R^T (X - t).  Coordinates
    get N(0, coord_noise_m) noise per component, and a fraction `outlier_fraction` of each object's pixels gets a coordinate drawn
    uniformly in the class's extent box.  The coordinates are then scaled into [0,1] by the extents
    (lib/gt_synthesize_layer/minibatch.py:605-616) into the class's three channels of a [B,H,W,3C] tensor, zero elsewhere.

    Returns make_refine_scene's dict (label, depth, meta, points, poses [N,9]: every placed object) plus
      coords  [B,H,W,3] f32  unscaled object coordinate of the labelled object (zero on the background)
      vertex  [B,H,W,3C] f32 scaled coordinates
      extents [C,3] f32"""
    C = num_classes
    sc = make_refine_scene(batch=batch, height=height, width=width, num_classes=C, objects_per_image=objects_per_image, seed=seed,
                           factor_depth=factor_depth, min_pixels=1)
    K = intrinsics(height, width)
    fx, fy, px, py = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    ext = extents_for(C)
    vv, uu = np.mgrid[0:height, 0:width].astype(np.float64)
    coords = np.zeros((batch, height, width, 3), np.float32)
    vertex = np.zeros((batch, height, width, 3 * C), np.float32)
    for row in sc["poses"]:
        b, cls = int(row[0]), int(row[1])
        R, t = quat_to_rot(row[2:6]), row[6:9]
        mask = sc["label"][b] == cls
        z = sc["depth"][b][mask].astype(np.float64) / factor_depth
        X = np.stack([(uu[mask] - px) / fx * z, (vv[mask] - py) / fy * z, z], -1)
        obj = (X - t) @ R
        rng = np.random.default_rng(seed + 7919 * b + cls)
        if coord_noise_m > 0:
            obj = obj + rng.normal(0.0, coord_noise_m, obj.shape)
        if outlier_fraction > 0:
            bad = rng.random(obj.shape[0]) < outlier_fraction
            obj[bad] = (rng.random((int(bad.sum()), 3)) - 0.5) * ext[cls]
        coords[b][mask] = obj
        vmin, vmax = -ext[cls].astype(np.float64) / 2, ext[cls].astype(np.float64) / 2
        vertex[b][mask, 3 * cls:3 * cls + 3] = (obj - vmin) / (vmax - vmin)
    sc.update(coords=coords, vertex=vertex, extents=ext)
    return sc


def make_pose_batch(num_rois: int, num_classes: int = 22, seed: int = 11, noise: float = 0.15):
    """prediction/target/weight [N,4C] for Averagedistance (vgg16_convs.py:195-200)."""
    rng = np.random.default_rng(seed)
    pred = np.zeros((num_rois, 4 * num_classes), dtype=np.float32)
    targ = np.zeros_like(pred)
    wt = np.zeros_like(pred)
    for n in range(num_rois):
        if n % 7 == 6:
            continue  # a ROI without a matched gt: all-zero weights
        c = int(rng.integers(1, num_classes))
        q = _rand_quat(rng)
        p = q + rng.normal(0, noise, 4)
        p /= np.linalg.norm(p)
        targ[n, 4 * c : 4 * c + 4] = q
        pred[n, 4 * c : 4 * c + 4] = p
        wt[n, 4 * c : 4 * c + 4] = 1
    return pred, targ, wt


def make_rois(num_rois: int, batch: int, height: int = 480, width: int = 640, num_classes: int = 22, seed: int = 5):
    """[N,7] ROI rows [b, cls, x1,y1,x2,y2, score] (SURVEY §8(d): w,h ~ U[40,240])."""
    rng = np.random.default_rng(seed)
    rois = np.zeros((num_rois, 7), dtype=np.float32)
    for n in range(num_rois):
        w = rng.uniform(40, 240) * width / 640.0
        h = rng.uniform(40, 240) * height / 480.0
        x1 = rng.uniform(-20, width - w + 20)
        y1 = rng.uniform(-20, height - h + 20)
        rois[n] = [rng.integers(0, batch), rng.integers(1, num_classes), x1, y1, x1 + w, y1 + h, rng.uniform(0, 500)]
    return rois


def make_projection_case(batch: int, height: int, width: int, channels: int, num_classes: int,
                         grid_size: int, seed: int = 3):
    """Inputs for Backproject / Project: feature map, label map, depth, meta (with a small
    rigid motion), 3-D label grid and a voxel feature grid.  The voxel grid covers
    x,y in [-3,3], z in [-3,4] (lib/fcn/test.py:1180), so depth in [0.5, 2.0] m lands inside."""
    rng = np.random.default_rng(seed)
    K = intrinsics(height, width)
    data = rng.standard_normal((batch, height, width, channels), dtype=np.float32)
    lab = rng.random((batch, height, width, num_classes), dtype=np.float32)
    depth = rng.uniform(0.5, 2.0, (batch, height, width, 1)).astype(np.float32)
    meta = np.zeros((batch, 1, 1, 48), dtype=np.float32)
    for b in range(batch):
        ang = rng.uniform(-0.05, 0.05, 3)
        cx, sx = np.cos(ang[0]), np.sin(ang[0])
        cy, sy = np.cos(ang[1]), np.sin(ang[1])
        cz, sz = np.cos(ang[2]), np.sin(ang[2])
        R = (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
             @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))
        t = rng.uniform(-0.05, 0.05, (3, 1))
        meta[b, 0, 0] = make_meta(K, grid_size, np.hstack([R, t]))
    label_3d = rng.random((batch, grid_size, grid_size, grid_size, num_classes), dtype=np.float32)
    vox = rng.standard_normal((batch, grid_size, grid_size, grid_size, channels), dtype=np.float32)
    return dict(data=data, label=lab, depth=depth, meta=meta, label_3d=label_3d, vox=vox)


def make_images(batch: int, height: int = 480, width: int = 640, seed: int = 21):
    """Uniform uint8 BGR images and depth (metres) for the full-network bench."""
    rng = np.random.default_rng(seed)
    rgb = rng.integers(0, 256, (batch, height, width, 3), dtype=np.uint8)
    depth = rng.uniform(0.5, 2.0, (batch, height, width)).astype(np.float32)
    return rgb, depth
