"""Float64 numpy restatement of the device pose refiner (DESIGN.md §12, csrc/pose_refine.cu), line for line.

Per ROI row: stage 1 re-centres the translation along its ray on the depth inliers (poses_refined); stage 2 runs projective
point-to-plane Gauss-Newton from 8 depth hypotheses; stage 3 scores each with the distinct-nearest-pixel metric and keeps the
first maximum (poses_icp).  Everything here is float64; the device forms the Gauss-Newton terms in fp64 and searches the score
window in fp32.
"""
from __future__ import annotations

import math

import numpy as np

DZ = (0.0, -0.02, -0.01, 0.01, 0.02, 0.03, 0.04, 0.05)   # depth hypotheses, in the reference's order
NUM_HYP = len(DZ)
RAY_NORMAL_MIN = 0.1      # -ray . n >= 0.1
SCORE_RADIUS = 0.01       # nearest-neighbour radius of the score (1 cm)
MIN_INLIERS = 6
PIVOT_REL = 1e-12
VIS_POINTS_PER_CELL = 8.0   # visibility grid: mean table points per cell of the projected bounding box
VIS_MAX_CELLS = 64          # at most 64 cells along either side of the grid
VIS_MARGIN = 0.003          # a point is visible within 3 mm of the front-most point of its cell
GATE_REL = 1e-5           # near-gate band of near_gate_count (relative to the size of the compared quantities)


# ---------------------------------------------------------------------------------------------------------------- geometry
def quat_normalize(q):
    q = np.asarray(q, dtype=np.float64)
    n = math.sqrt(float(np.dot(q, q)))
    return np.array([1.0, 0.0, 0.0, 0.0]) if n == 0.0 else q / n


def quat_to_rot(q):
    """(w, x, y, z), normalised first -> 3x3."""
    w, x, y, z = quat_normalize(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def quat_mul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])


def se3_exp(xi):
    """Sophus SE3::exp of xi = (upsilon, omega): quaternion of exp(omega^) and V upsilon."""
    xi = np.asarray(xi, dtype=np.float64)
    ups, w = xi[:3], xi[3:]
    th2 = float(np.dot(w, w))
    th = math.sqrt(th2)
    if th < 1e-4:
        k, B, Cc = 0.5 - th2 / 48.0, 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    else:
        k, B, Cc = math.sin(0.5 * th) / th, (1.0 - math.cos(th)) / th2, (th - math.sin(th)) / (th2 * th)
    dq = np.array([math.cos(0.5 * th), k * w[0], k * w[1], k * w[2]])
    wxu = np.cross(w, ups)
    dt = ups + B * wxu + Cc * np.cross(w, wxu)
    return dq, dt


def apply_update(q, t, xi):
    """T <- exp(xi) T, quaternion renormalised."""
    dq, dt = se3_exp(xi)
    qn = quat_normalize(quat_mul(dq, q))
    tn = quat_to_rot(dq) @ np.asarray(t, np.float64) + dt
    return qn, tn


def ldlt_solve(A, g):
    """LDL^T of the symmetric 6x6 A; None when a pivot is <= 1e-12 trace(A)."""
    n = 6
    thr = PIVOT_REL * float(np.trace(A))
    L = np.eye(n)
    d = np.zeros(n)
    for j in range(n):
        dj = A[j, j] - sum(L[j, k] * L[j, k] * d[k] for k in range(j))
        if not dj > thr:
            return None
        d[j] = dj
        for i in range(j + 1, n):
            L[i, j] = (A[i, j] - sum(L[i, k] * L[j, k] * d[k] for k in range(j))) / dj
    y = np.zeros(n)
    for i in range(n):
        y[i] = g[i] - sum(L[i, k] * y[k] for k in range(i))
    z = y / d
    x = np.zeros(n)
    for i in reversed(range(n)):
        x[i] = z[i] - sum(L[k, i] * x[k] for k in range(i + 1, n))
    return x


# ---------------------------------------------------------------------------------------------------------------- live data
class Live:
    """Vertices and normals of one image's depth, masked to class c."""

    def __init__(self, label, depth, c, fx, fy, px, py, factor, znear, zfar):
        H, W = label.shape
        self.H, self.W, self.fx, self.fy, self.px, self.py = H, W, fx, fy, px, py
        self.znear, self.zfar = znear, zfar
        z = np.asarray(depth, np.float64) / factor
        self.valid = (label == c) & (z > znear) & (z < zfar)
        vv, uu = np.mgrid[0:H, 0:W].astype(np.float64)
        self.X = np.stack([(uu - px) * z / fx, (vv - py) * z / fy, z], -1)
        n = np.zeros((H, W, 3))
        nvalid = np.zeros((H, W), bool)
        v4 = (self.valid[1:-1, 1:-1] & self.valid[1:-1, 2:] & self.valid[1:-1, :-2] & self.valid[2:, 1:-1] & self.valid[:-2, 1:-1])
        cr = np.cross(self.X[1:-1, 2:] - self.X[1:-1, :-2], self.X[2:, 1:-1] - self.X[:-2, 1:-1])
        ln = np.linalg.norm(cr, axis=-1)
        ok = v4 & (ln > 0)
        cr = cr / np.where(ln > 0, ln, 1.0)[..., None]
        flip = np.sum(cr * self.X[1:-1, 1:-1], -1) > 0
        cr[flip] = -cr[flip]
        n[1:-1, 1:-1] = cr
        nvalid[1:-1, 1:-1] = ok
        self.n, self.nvalid = n, nvalid


def visible(live: Live, Q):
    """Self-occlusion of the model, standing in for the reference's render: the points in the depth range are binned by their
    projection (fx q_x / q_z + px, fy q_y / q_z + py) into square cells over their bounding box, side
    s = max(sqrt(VIS_POINTS_PER_CELL * bw * bh / P), max(bw, bh) / VIS_MAX_CELLS, 1) pixels; a point is visible iff its
    q_z <= (the smallest q_z of its cell) + VIS_MARGIN."""
    P = Q.shape[0]
    inz = (Q[:, 2] > live.znear) & (Q[:, 2] < live.zfar)
    vis = np.zeros(P, bool)
    if not inz.any():
        return vis
    zs = np.where(inz, Q[:, 2], 1.0)
    fu = live.fx * Q[:, 0] / zs + live.px
    fv = live.fy * Q[:, 1] / zs + live.py
    u0, u1 = fu[inz].min(), fu[inz].max()
    v0, v1 = fv[inz].min(), fv[inz].max()
    bw, bh = u1 - u0, v1 - v0
    side = max(math.sqrt(VIS_POINTS_PER_CELL * bw * bh / P), max(bw, bh) / VIS_MAX_CELLS, 1.0)
    gw = int((bw / side)) + 1
    cell = np.where(inz, np.trunc((fv - v0) / side) * gw + np.trunc((fu - u0) / side), 0).astype(np.int64)
    zmin = np.full(gw * (int(bh / side) + 1), np.inf)
    np.minimum.at(zmin, cell[inz], Q[inz, 2])
    vis[inz] = Q[inz, 2] <= zmin[cell[inz]] + VIS_MARGIN
    return vis


def associate(live: Live, pts, q, t, max_error):
    """Projective association of the model points under (q, t).  Returns a dict with the inlier mask and, per point, the
    transformed point, live vertex, normal and point-to-plane error (meaningful where inlier)."""
    R = quat_to_rot(q)
    Q = pts.astype(np.float64) @ R.T + np.asarray(t, np.float64)
    P = Q.shape[0]
    inz = (Q[:, 2] > live.znear) & (Q[:, 2] < live.zfar)
    zs = np.where(inz, Q[:, 2], 1.0)
    fu = live.fx * Q[:, 0] / zs + live.px + 0.5
    fv = live.fy * Q[:, 1] / zs + live.py + 0.5
    inb = inz & (fu >= 3) & (fu < live.W - 3) & (fv >= 3) & (fv < live.H - 3)
    u = np.where(inb, np.trunc(np.where(inb, fu, 0)), 0).astype(np.int64)
    v = np.where(inb, np.trunc(np.where(inb, fv, 0)), 0).astype(np.int64)
    ok = inb & live.nvalid[v, u] & visible(live, Q)
    X = live.X[v, u]
    n = live.n[v, u]
    qn = np.linalg.norm(Q, axis=1)
    ray = -np.sum(Q * n, 1) / np.where(qn > 0, qn, 1.0)
    ok &= ray >= RAY_NORMAL_MIN
    e = np.sum(n * (X - Q), 1)
    inl = ok & (np.abs(e) <= max_error)
    return dict(inlier=inl, Q=Q, X=X, n=n, e=e, fu=fu, fv=fv, ray=ray, ok_before_e=ok, inz=inz, P=P)


def near_gate_count(live: Live, a, max_error):
    """Points whose association decision sits within GATE_REL of a gate: the depth range, the rounding of the projection, the
    ray / normal test and |e| <= max_error.  Any other arithmetic may decide them differently."""
    Q = a["Q"]
    qn = np.linalg.norm(Q, axis=1)
    near = (np.abs(Q[:, 2] - live.znear) <= GATE_REL * live.zfar) | (np.abs(Q[:, 2] - live.zfar) <= GATE_REL * live.zfar)
    for f in (a["fu"], a["fv"]):
        near |= a["inz"] & (np.abs(f - np.round(f)) <= GATE_REL * np.abs(f) + 1e-9)
    near |= a["inz"] & (np.abs(a["ray"] - RAY_NORMAL_MIN) <= GATE_REL)
    near |= a["ok_before_e"] & (np.abs(np.abs(a["e"]) - max_error) <= GATE_REL * np.maximum(qn, max_error))
    return int(near.sum())


def gauss_newton_system(a):
    """A = sum J^T J, g = sum J^T e_w over the inliers, J = w n^T [I | -[q]x] = w [n, q x n], w = 1 / X_z."""
    m = a["inlier"]
    Q, X, n, e = a["Q"][m], a["X"][m], a["n"][m], a["e"][m]
    w = 1.0 / X[:, 2]
    J = w[:, None] * np.concatenate([n, np.cross(Q, n)], 1)
    return J.T @ J, J.T @ (w * e), int(m.sum())


def gn_step(live, pts, q, t, max_error):
    """One Gauss-Newton step from (q, t): (new q, new t, inliers at (q, t), stopped)."""
    a = associate(live, pts, q, t, max_error)
    A, g, n = gauss_newton_system(a)
    if n < MIN_INLIERS:
        return q, t, n, True
    xi = ldlt_solve(A, g)
    if xi is None:
        return q, t, n, True
    qn, tn = apply_update(q, t, xi)
    return qn, tn, n, False


def score(live: Live, pts, q, t):
    """#distinct nearest live pixels within 1 cm of a transformed model point / P, searched in the projective window."""
    R = quat_to_rot(q)
    Q = pts.astype(np.float64) @ R.T + np.asarray(t, np.float64)
    P = Q.shape[0]
    H, W = live.H, live.W
    sel = np.full(P, -1, np.int64)
    for i in range(P):
        qz = Q[i, 2]
        if not (live.znear < qz < live.zfar):
            continue
        fu = live.fx * Q[i, 0] / qz + live.px + 0.5
        fv = live.fy * Q[i, 1] / qz + live.py + 0.5
        if not (fu >= 0 and fu < W and fv >= 0 and fv < H):
            continue
        u, v = int(fu), int(fv)
        k = int(math.ceil(SCORE_RADIUS * live.fx / max(qz - SCORE_RADIUS, live.znear)))
        v0, v1, u0, u1 = max(v - k, 0), min(v + k, H - 1), max(u - k, 0), min(u + k, W - 1)
        Xw = live.X[v0:v1 + 1, u0:u1 + 1]
        d2 = np.sum((Xw - Q[i]) ** 2, -1)
        d2 = np.where(live.valid[v0:v1 + 1, u0:u1 + 1] & (d2 < SCORE_RADIUS * SCORE_RADIUS), d2, np.inf)
        j = int(np.argmin(d2))              # row-major = ascending flat index: ties go to the lowest
        if np.isfinite(d2.flat[j]):
            sel[i] = (v0 + j // (u1 - u0 + 1)) * W + (u0 + j % (u1 - u0 + 1))
    s = sel[sel >= 0]
    return int(np.unique(s).size), P


def stage1(live, pts, q, t, max_error):
    """Depth re-centring along the ray on the inliers at the input pose."""
    q = quat_normalize(q)
    t = np.asarray(t, np.float64)
    a = associate(live, pts, q, t, max_error)
    m = a["inlier"]
    if not m.any():
        return q, t.copy()
    delta = float(np.mean(a["X"][m, 2] - a["Q"][m, 2]))
    tz = t[2] + delta
    rx, ry = (0.0, 0.0) if t[2] == 0 else (t[0] / t[2], t[1] / t[2])
    return q, np.array([rx * tz, ry * tz, tz])


def refine_row(label, depth, meta, roi, pose, points, batch_offset=0, factor=10000.0, znear=0.25, zfar=6.0, max_error=0.01,
               min_pixels=400, iterations=8):
    """One ROI row.  label [B,H,W], depth [B,H,W] raw, meta [B,>=6].  Returns (refined [7], icp [7], info [4], trace
    [8, iterations + 1, 8]); a skipped row is all zero except info[0] = n_mask."""
    B = label.shape[0]
    C = points.shape[0]
    b, c = int(roi[0]) - batch_offset, int(roi[1])
    z7 = np.zeros(7)
    trace = np.zeros((NUM_HYP, iterations + 1, 8))
    if not (0 < c < C and 0 <= b < B):
        return z7, z7.copy(), np.zeros(4), trace
    n_mask = int((label[b] == c).sum())
    if n_mask < min_pixels:
        return z7, z7.copy(), np.array([n_mask, 0, 0, 0], np.float64), trace
    m = np.asarray(meta[b], np.float64).reshape(-1)
    live = Live(label[b], depth[b], c, m[0], m[4], m[2], m[5], factor, znear, zfar)
    pts = points[c]
    q1, t1 = stage1(live, pts, pose[:4], pose[4:7], max_error)
    best = (-1, 0, None, None, 0)
    for h in range(NUM_HYP):
        q, t = q1.copy(), t1 + np.array([0.0, 0.0, DZ[h]])
        s = 0
        while s < iterations:
            qn, tn, n, stop = gn_step(live, pts, q, t, max_error)
            trace[h, s] = np.r_[q, t, n]
            s += 1
            if stop:
                s -= 1
                break
            q, t = qn, tn
        nfin = int(associate(live, pts, q, t, max_error)["inlier"].sum())
        for k in range(s, iterations + 1):
            trace[h, k] = np.r_[q, t, nfin]
        cnt, P = score(live, pts, q, t)
        if cnt > best[0]:
            best = (cnt, h, q, t, nfin)
    cnt, h, q, t, nfin = best
    info = np.array([n_mask, h, cnt / points.shape[1], nfin], np.float64)
    return np.r_[q1, t1], np.r_[q, t], info, trace


def refine(label, depth, meta, rois, poses, points, num_rows=None, batch_offset=0, **kw):
    """The batched call: capacity-shaped outputs, rows >= num_rows zero."""
    cap = rois.shape[0]
    it = kw.get("iterations", 8)
    meta = np.asarray(meta, np.float32).reshape(label.shape[0], -1)
    out = dict(poses_refined=np.zeros((cap, 7)), poses_icp=np.zeros((cap, 7)), icp_info=np.zeros((cap, 4)),
               icp_trace=np.zeros((cap, NUM_HYP, it + 1, 8)))
    n = cap if num_rows is None else min(int(num_rows), cap)
    for r in range(n):
        a, b_, c_, d_ = refine_row(label, depth, meta, rois[r], poses[r], points, batch_offset, **kw)
        out["poses_refined"][r], out["poses_icp"][r], out["icp_info"][r], out["icp_trace"][r] = a, b_, c_, d_
    return out
