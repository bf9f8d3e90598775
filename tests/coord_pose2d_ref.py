"""float64 restatement of the colour-only object-coordinate estimator (csrc/coord_pose.cu k_sample2d / k_ransac<true>, DESIGN.md
§13), the tests' oracle.

It follows Synthesizer::estimatePose2D (lib/synthesize/synthesize.cpp:1571-1767) as written, with the device's random streams and
its P3P (Grunert's quartic, the roots bisected as the device does, Kabsch on the three camera points).  The survivor keeps its P3P
pose: the reference's refit (updateHyp3D on an empty 3-D inlier list) returns at once and its Nelder-Mead energy is not finite.
Shared pieces (Philox words, object coordinates, Kabsch, the projected-box area, the subset rule) come from tests/coord_pose_ref.py.
"""
from __future__ import annotations

import math

import numpy as np

from tests import coord_pose_ref as ref

F32 = np.float32
GATE_2D = 10.0          # inlierThreshold2D = minDist2D (px)
BISECT = 200


def ctr_p2a(h, att):
    return (4 << 60) | (h << 32) | att


def ctr_p2b(h, att):
    return (5 << 60) | (h << 32) | att


def horner(c, x):
    v = c[0]
    for a in c[1:]:
        v = v * x + a
    return v


def bisect(c, lo, hi, flo):
    mid = 0.5 * (lo + hi)
    for _ in range(BISECT):
        if not (lo < mid < hi):
            break
        fm = horner(c, mid)
        if fm == 0.0:
            return mid
        if (fm < 0.0) == (flo < 0.0):
            lo, flo = mid, fm
        else:
            hi = mid
        mid = 0.5 * (lo + hi)
    return mid


def quartic_roots(p):
    """Real roots of x^4 + p0 x^3 + p1 x^2 + p2 x + p3, ascending: derivative roots bracket, bisection to the last bit."""
    bound = max([1.0] + [1.0 + abs(a) for a in p])
    polys = [[6.0, 3.0 * p[0], p[1]], [4.0, 3.0 * p[0], 2.0 * p[1], p[2]], [1.0, p[0], p[1], p[2], p[3]]]
    r = [-p[0] / 4.0]
    for c in polys:
        nr, lo = [], -bound
        flo = horner(c, lo)
        for i in range(len(r) + 1):
            hi = min(max(r[i], -bound), bound) if i < len(r) else bound
            fhi = horner(c, hi)
            if flo != 0.0 and fhi != 0.0 and (flo < 0.0) != (fhi < 0.0) and lo < hi:
                nr.append(bisect(c, lo, hi, flo))
            lo, flo = hi, fhi
        r = nr
    return r


def project(R, t, cam, X):
    """cv::projectPoints of one point (double): (u, v)."""
    fx, fy, px, py = cam
    q = R @ np.asarray(X, np.float64) + t
    iz = 1.0 / q[2] if q[2] != 0 else 1.0
    return q[0] * iz * fx + px, q[1] * iz * fy + py


def p3p(obj, pu, pv, cam):
    """P3P on the first three (object point, pixel) pairs by Grunert's quartic; the root whose pose reprojects the fourth pair
    closest wins (first on a tie).  obj [4,3] float32 values, pu / pv the pixel coordinates.  (R, t) or None.  Scalar Python
    floats, so every operation rounds on its own in the written order, as on the device."""
    fx, fy, px, py = cam
    f, P = [], [[float(x) for x in o] for o in obj[:3]]
    for k in range(3):
        xn, yn = (float(pu[k]) - px) / fx, (float(pv[k]) - py) / fy
        nn = math.sqrt(xn * xn + yn * yn + 1.0)
        f.append((xn / nn, yn / nn, 1.0 / nn))

    def sq(i, j):
        dx, dy, dz = P[i][0] - P[j][0], P[i][1] - P[j][1], P[i][2] - P[j][2]
        return dx * dx + dy * dy + dz * dz

    dot = lambda i, j: f[i][0] * f[j][0] + f[i][1] * f[j][1] + f[i][2] * f[j][2]
    a2, b2, c2 = sq(1, 2), sq(0, 2), sq(0, 1)
    if not b2 > 0:
        return None
    ca, cb, cg = dot(1, 2), dot(0, 2), dot(0, 1)
    amc, apc = (a2 - c2) / b2, (a2 + c2) / b2
    A4 = (amc - 1.0) * (amc - 1.0) - 4.0 * c2 / b2 * ca * ca
    A3 = 4.0 * (amc * (1.0 - amc) * cb - (1.0 - apc) * ca * cg + 2.0 * c2 / b2 * ca * ca * cb)
    A2 = 2.0 * (amc * amc - 1.0 + 2.0 * amc * amc * cb * cb + 2.0 * (b2 - c2) / b2 * ca * ca - 4.0 * apc * ca * cb * cg +
                2.0 * (b2 - a2) / b2 * cg * cg)
    A1 = 4.0 * (-amc * (1.0 + amc) * cb + 2.0 * a2 / b2 * cg * cg * cb - (1.0 - apc) * ca * cg)
    A0 = (1.0 + amc) * (1.0 + amc) - 4.0 * a2 / b2 * cg * cg
    if A4 == 0:
        return None
    p = [A3 / A4, A2 / A4, A1 / A4, A0 / A4]
    if not all(math.isfinite(x) for x in p):
        return None
    best, out = math.inf, None
    for v in quartic_roots(p):
        den = 2.0 * (cg - v * ca)
        if not v > 0 or den == 0:
            continue
        u = ((amc - 1.0) * v * v - 2.0 * amc * cb * v + 1.0 + amc) / den
        s1q = b2 / (1.0 + v * v - 2.0 * v * cb)
        if not (u > 0 and s1q > 0 and math.isfinite(s1q)):
            continue
        s1 = math.sqrt(s1q)
        X = np.array([[s1 * x for x in f[0]], [u * s1 * x for x in f[1]], [v * s1 * x for x in f[2]]])
        sol = ref.kabsch(np.array(P), X)
        if sol is None:
            continue
        q = project(*sol, cam, obj[3])
        err = math.sqrt((float(pu[3]) - q[0]) ** 2 + (float(pv[3]) - q[1]) ** 2)
        if err < best:
            best, out = err, sol
    return out


def line_dist(p, q, r):
    """pointLineDistance: float differences and cross product, double norms (NaN for coincident p, q)."""
    a, b = (q - p).astype(F32), (r - p).astype(F32)
    c = np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]], F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.sqrt(np.sum(c.astype(np.float64) ** 2)) / np.sqrt(np.sum(a.astype(np.float64) ** 2))


def attempt(vertex, ext, cam, W, H, key, lists, objs, h, att):
    """One attempt: (accepted, obj, four pixels, R, t)."""
    w0, w1 = ref.words(key, ctr_p2a(h, att)), ref.words(key, ctr_p2b(h, att))
    obj = objs[ref.uniform_int(w0[0], len(objs))]
    L = lists[obj]
    pix, pts, ocs = [], [], []
    for k in range(4):
        idx = int(L[ref.uniform_int(w0[k + 1] if k < 3 else w1[0], len(L))])
        pt = np.array([idx % W, idx // W], F32)
        pix.append(idx)
        ds = [math.sqrt(float(d[0]) ** 2 + float(d[1]) ** 2) for d in (p - pt for p in pts)]
        if ds and 0 < min(ds) < GATE_2D:
            return False, obj, pix, None, None
        o = ref.mode_at(vertex, ext, obj, idx)
        if not o.any():
            return False, obj, pix, None, None
        ds = [ref.dist_f(p, o) for p in ocs]
        if ds and 0 < min(ds) < ref.GATE:
            return False, obj, pix, None, None
        pts.append(pt), ocs.append(o)
    for i, j, k in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)):
        if line_dist(ocs[i], ocs[j], ocs[k]) < ref.GATE:      # NaN does not reject
            return False, obj, pix, None, None
    pu, pv = [p[0] for p in pts], [p[1] for p in pts]
    sol = p3p(ocs, pu, pv, cam)
    if sol is None:
        return False, obj, pix, None, None
    R, t = sol
    for k in range(4):
        q = project(R, t, cam, ocs[k])
        dx, dy = F32(pu[k] - F32(q[0])), F32(pv[k] - F32(q[1]))
        if not math.sqrt(float(dx) ** 2 + float(dy) ** 2) < GATE_2D:
            return False, obj, pix, None, None
    if ref.bb_area(ext[obj], R, t, *(F32(x) for x in cam), W, H) < ref.MIN_AREA:
        return False, obj, pix, None, None
    return True, obj, pix, R, t


def sample(vertex, ext, cam, W, H, key, lists, C):
    """The 256 hypotheses of one image: dicts (obj, attempts, pix, R, t) (obj = 0: none)."""
    counts = [len(l) for l in lists]
    objs = [c for c in range(1, C) if counts[c] > ref.MIN_AREA]
    hyps = []
    for h in range(ref.NUM_HYP):
        res = dict(obj=0, attempts=ref.MAX_ATTEMPTS if objs else 0, pix=[-1] * 4, R=None, t=None)
        for att in range(ref.MAX_ATTEMPTS if objs else 0):
            ok, obj, pix, R, t = attempt(vertex, ext, cam, W, H, key, lists, objs, h, att)
            if ok:
                res.update(obj=obj, attempts=att + 1, pix=pix, R=R, t=t)
                break
        hyps.append(res)
    return hyps


def reprojection_distance(R, t, cam, obj, pix_uv):
    """countInliers2D's distance of every (object point, pixel) pair, double."""
    fx, fy, px, py = cam
    q = obj.astype(np.float64) @ R.T + t
    iz = np.where(q[:, 2] != 0, 1.0 / np.where(q[:, 2] != 0, q[:, 2], 1.0), 1.0)
    u, v = q[:, 0] * iz * fx + px, q[:, 1] * iz * fy + py
    return np.sqrt((pix_uv[:, 0] - u) ** 2 + (pix_uv[:, 1] - v) ** 2)


def estimate_image(label, vertex, ext, cam, key, C):
    """One image; cam = (fx, fy, px, py).  Returns poses [C,3,4], info [C,6] and traces (hyps, per class the per-round dicts)."""
    H, W = label.shape
    cam = tuple(float(F32(x)) for x in cam)
    lists = ref.pixel_lists(label, np.ones_like(label, np.float32), C)
    hyps = sample(vertex, ext, cam, W, H, key, lists, C)
    exhausted = sum(1 for h in hyps if h["obj"] == 0 and h["attempts"] == ref.MAX_ATTEMPTS)
    poses = np.zeros((C, 3, 4))
    info = np.zeros((C, 6))
    rounds = {}
    for c in range(C):
        N = len(lists[c])
        ids = [h for h in range(ref.NUM_HYP) if c > 0 and N > ref.MIN_AREA and hyps[h]["obj"] == c]
        info[c] = (N if c else 0, len(ids), 0, -1, exhausted if c else 0, -1)
        if not ids:
            continue
        L = lists[c]
        tr = []
        for r in range(ref.ROUNDS):
            pix = L[ref.subset(L, c, r, key)]
            uv = np.stack([pix % W, pix // W], 1).astype(np.float64)
            obj = np.array([ref.mode_at(vertex, ext, c, i) for i in pix], F32).reshape(-1, 3)
            cnt, near = {}, {}
            for h in ids:
                d = reprojection_distance(hyps[h]["R"], hyps[h]["t"], cam, obj, uv)
                cnt[h] = int(np.sum(d < GATE_2D))
                near[h] = int(np.sum(np.abs(d - GATE_2D) <= 1e-6 * GATE_2D))
            order = sorted(ids, key=lambda h: (-cnt[h], h))
            ids = order[:len(ids) // 2 if len(ids) > 1 else len(ids)]
            tr.append(dict(taken=len(pix), hash=int(pix.sum()) & 0xFFFFFFFF, counts=cnt, near=near, best=ids[0], best_count=cnt[ids[0]],
                           subset=pix))
        rounds[c] = tr
        h = ids[0]
        poses[c, :, :3], poses[c, :, 3] = hyps[h]["R"], hyps[h]["t"]
        info[c, 2], info[c, 5] = tr[-1]["best_count"], h
    return dict(poses=poses, info=info, hyps=hyps, rounds=rounds, lists=lists)
