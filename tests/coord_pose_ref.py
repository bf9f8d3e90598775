"""float64 numpy restatement of the object-coordinate pose estimator (csrc/coord_pose.cu, DESIGN.md §13), the tests' oracle.

It follows Synthesizer::estimatePose3D (lib/synthesize/synthesize.cpp:1769-1966) step by step with the device's random streams
(Philox4x32-10, tests/augment_ref.philox4x32_10) and returns per-image traces: hypotheses (class, attempts, pixel triple, pose),
per-round subsets, counts and survivors, and the final poses.  The SVD is numpy's; the reductions are sequential.
"""
from __future__ import annotations

import numpy as np

from tests.augment_ref import philox4x32_10

F32 = np.float32
NUM_HYP, ROUNDS, BATCH, MAX_INL, MIN_FINAL, MIN_AREA = 256, 8, 1000, 1000, 10, 400
MAX_TAKEN, MAX_ATTEMPTS, NM_EVALS, RANK_TOL = 12288, 1024, 100, 1e-6
GATE = float(np.float32(0.01))
HOLE = 0x80000000


def words(key, ctr):
    return [int(x[0]) for x in philox4x32_10(int(key), np.array([ctr], np.uint64))]


def uniform_int(w, n):
    return (int(w) * int(n)) >> 32


def ctr_hyp(h, att):
    return (1 << 60) | (h << 32) | att


def ctr_sub(c, r, k):
    return (2 << 60) | (c << 48) | (r << 40) | k


def ctr_fil(h, r, j):
    return (3 << 60) | (h << 48) | (r << 40) | j


def pixel_lists(label, depth, C):
    """Per class the pixel indices in column-major order (x outer, y inner), hole flag in bit 31."""
    H, W = label.shape
    lt, dt = label.T.reshape(-1), depth.T.reshape(-1)
    idx = (np.arange(H)[None, :] * W + np.arange(W)[:, None]).reshape(-1)
    return [(idx[lt == c] | np.where(dt[lt == c] == 0, HOLE, 0)).astype(np.int64) for c in range(C)]


def eye_at(depth, W, fx, fy, px, py, factor, idx):
    x, y, d = F32(idx % W), F32(idx // W), F32(depth.reshape(-1)[idx])
    return np.array([(x - F32(px)) * d / F32(fx) / F32(factor), (y - F32(py)) * d / F32(fy) / F32(factor), d / F32(factor)], F32)


def mode_at(vertex, ext, c, idx):
    v = vertex.reshape(-1, vertex.shape[-1])[idx, 3 * c:3 * c + 3].astype(F32)
    e = ext[c].astype(F32)
    vmin, vmax = -e / F32(2), e / F32(2)
    den = vmax - vmin
    with np.errstate(divide="ignore", invalid="ignore"):
        a = (1.0 / den.astype(np.float64)).astype(F32)
        b = (-1.0 * vmin.astype(np.float64) / den.astype(np.float64)).astype(F32)
        return ((v - b) / a).astype(F32)


def dist_f(p, q):
    d = (p - q).astype(np.float64)
    return float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]))


def kabsch(A, Bp):
    """Hypothesis::calcRigidBodyTransform on pairs A (object) -> B (camera), [n,3] float64; None when of rank < 2."""
    cA, cB = A.sum(0) * (1.0 / len(A)), Bp.sum(0) * (1.0 / len(Bp))
    a = (A - cA).T @ (Bp - cB)
    u, s, vt = np.linalg.svd(a)
    if not (s[0] > 0 and s[1] > RANK_TOL * s[0] and np.isfinite(s[0])):
        return None
    v = vt.T
    d = -1.0 if np.linalg.det(v @ u.T) < 0 else 1.0
    R = v @ np.diag([1.0, 1.0, d]) @ u.T
    return R, cB - R @ cA


def f2i(v):
    """`int = float` as compiled for x86-64 (cvttss2si): truncation, INT_MIN outside the int range."""
    v = float(np.float32(v))
    return int(v) if -2.0**31 <= v < 2.0**31 else -2**31


def bb_area(e, R, t, fx, fy, px, py, W, H):
    h = e.astype(F32) / F32(2)
    minX, maxX, minY, maxY = W - 1, 0, H - 1, 0
    for k in range(8):
        p = np.array([-h[0] if k & 4 else h[0], -h[1] if k & 2 else h[1], -h[2] if k & 1 else h[2]], np.float64)
        q = R @ p + t
        iz = 1.0 / q[2] if q[2] != 0 else 1.0
        u, v = F32(q[0] * iz * float(F32(fx)) + float(F32(px))), F32(q[1] * iz * float(F32(fy)) + float(F32(py)))
        minX = f2i(u if u < F32(minX) else F32(minX))
        minY = f2i(v if v < F32(minY) else F32(minY))
        maxX = f2i(u if F32(maxX) < u else F32(maxX))
        maxY = f2i(v if F32(maxY) < v else F32(maxY))
    cl = lambda x, hi: min(max(x, 0), hi)
    minX, maxX, minY, maxY = cl(minX, W - 1), cl(maxX, W - 1), cl(minY, H - 1), cl(maxY, H - 1)
    return (maxX - minX + 1) * (maxY - minY + 1)


def sample(label, depth, vertex, ext, cam, factor, key, lists, C):
    """The 256 hypotheses of one image: dicts (obj, attempts, pix, R, t) (obj = 0: none)."""
    H, W = label.shape
    fx, fy, px, py = cam
    counts = np.array([len(l) for l in lists])
    objs = [c for c in range(1, C) if counts[c] > MIN_AREA]
    hyps = []
    for h in range(NUM_HYP):
        res = dict(obj=0, attempts=0, pix=[-1, -1, -1], R=None, t=None)
        for att in range(MAX_ATTEMPTS if objs else 0):
            res["attempts"] = att + 1
            w = words(key, ctr_hyp(h, att))
            obj = objs[uniform_int(w[0], len(objs))]
            L = lists[obj]
            eyes, ocs, pix, ok = [], [], [], True
            for k in range(3):
                entry = int(L[uniform_int(w[k + 1], len(L))])
                if entry & HOLE:
                    ok = False
                    break
                e = eye_at(depth, W, fx, fy, px, py, factor, entry)
                ds = [dist_f(p, e) for p in eyes]
                if ds and 0 < min(ds) < GATE:
                    ok = False
                    break
                o = mode_at(vertex, ext, obj, entry)
                if not o.any():
                    ok = False
                    break
                ds = [dist_f(p, o) for p in ocs]
                if ds and 0 < min(ds) < GATE:
                    ok = False
                    break
                eyes.append(e), ocs.append(o), pix.append(entry)
            if not ok:
                continue
            A, Bp = np.array(ocs, np.float64), np.array(eyes, np.float64)
            sol = kabsch(A, Bp)
            if sol is None:
                continue
            R, t = sol
            if np.any(np.linalg.norm(Bp - (A @ R.T + t), axis=1) >= GATE):
                continue
            if bb_area(ext[obj], R, t, fx, fy, px, py, W, H) < MIN_AREA:
                continue
            res.update(obj=obj, pix=pix, R=R, t=t)
            break
        hyps.append(res)
    return hyps


def subset(L, c, r, key):
    """Pixel-list positions taken in round r (countInliers3D's stepping rule, one draw per taken pixel)."""
    N = len(L)
    p = F32(F32(BATCH * (r + 1)) / F32(N))
    all_ = not p < F32(1)
    lq = 0.0 if all_ else np.log1p(-float(p))
    hole = (L & HOLE) != 0
    out, pos, k = [], 0, 0
    while pos < N and len(out) < MAX_TAKEN:
        if hole[pos]:
            pos += 1
            continue
        out.append(pos)
        if all_:
            pos += 1
        else:
            w = words(key, ctr_sub(c, r, k))
            u = float((((w[0] << 32) | w[1]) >> 11) + 1) * 2.0**-53
            g = np.floor(np.log(u) / lq)
            pos += 1 if g < 1 else (N if g > N else int(g))
        k += 1
    return np.array(out, np.int64)


def rodrigues_exp(r):
    th = float(np.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]))
    if th < 2.220446049250313e-16:
        return np.eye(3)
    c, s, c1 = np.cos(th), np.sin(th), 1.0 - np.cos(th)
    x, y, z = r[0] / th, r[1] / th, r[2] / th
    return np.array([[c + c1 * x * x, c1 * x * y - s * z, c1 * x * z + s * y], [c1 * x * y + s * z, c + c1 * y * y, c1 * y * z - s * x],
                     [c1 * x * z - s * y, c1 * y * z + s * x, c + c1 * z * z]])


def rodrigues_log(R):
    rx, ry, rz = R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]
    s = np.sqrt((rx * rx + ry * ry + rz * rz) * 0.25)
    c = min(max((R[0, 0] + R[1, 1] + R[2, 2] - 1.0) * 0.5, -1.0), 1.0)
    th = np.arccos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        rx = np.sqrt(max((R[0, 0] + 1) * 0.5, 0.0))
        ry = np.sqrt(max((R[1, 1] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0)
        rz = np.sqrt(max((R[2, 2] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)
        if abs(rx) < abs(ry) and abs(rx) < abs(rz) and ((R[1, 2] > 0) != (ry * rz > 0)):
            rz = -rz
        th /= np.sqrt(rx * rx + ry * ry + rz * rz)
        return np.array([rx, ry, rz]) * th
    return np.array([rx, ry, rz]) * (th / (2.0 * s))


def energy(x, obj, eye):
    """optEnergy3D: rotation rounded to float, mean camera distance (sum in double, rounded to float)."""
    Rf = rodrigues_exp(x).astype(F32).astype(np.float64)
    q = (obj.astype(np.float64) @ Rf.T).astype(F32).astype(np.float64) + x[3:]
    q = q.astype(F32).astype(np.float64)
    d = np.sqrt(((q - eye.astype(np.float64)) ** 2).sum(1))
    return float(F32(F32(d.sum()) / F32(len(obj))))


def nelder_mead(x0, obj, eye):
    """The device's bounded Nelder-Mead (DESIGN §13)."""
    rr = 10.0 * 3.1415926 / 180.0
    rng = np.array([rr, rr, rr, 0.1, 0.1, 0.5])
    lb, ub = x0 - rng, x0 + rng
    clamp = lambda x: np.minimum(np.maximum(x, lb), ub)
    X = [x0.copy()] + [x0 + 0.5 * rng[i] * np.eye(6)[i] for i in range(6)]
    f = [energy(x, obj, eye) for x in X]
    ev = 7
    order = list(range(7))
    while ev < NM_EVALS:
        ordered = sorted(range(7), key=lambda v: (f[v], order.index(v)))
        order[:] = ordered
        wv = order[6]
        xc = sum(X[v] for v in order[:6]) / 6.0
        xr = clamp(xc + (xc - X[wv]))
        fr = energy(xr, obj, eye)
        ev += 1
        if fr < f[order[0]]:
            xt, flag = clamp(xc + 2.0 * (xc - X[wv])), 1
        elif fr < f[order[5]]:
            X[wv], f[wv] = xr, fr
            continue
        elif fr < f[wv]:
            xt, flag = clamp(xc + 0.5 * (xr - xc)), 2
        else:
            xt, flag = clamp(xc + 0.5 * (X[wv] - xc)), 3
        if ev >= NM_EVALS:
            if flag == 1:
                X[wv], f[wv] = xr, fr
            break
        ft = energy(xt, obj, eye)
        ev += 1
        if flag == 1:
            X[wv], f[wv] = (xt, ft) if ft < fr else (xr, fr)
        elif (ft <= fr) if flag == 2 else (ft < f[wv]):
            X[wv], f[wv] = xt, ft
        else:
            for k in range(1, 7):
                if ev >= NM_EVALS:
                    break
                v, bv = order[k], order[0]
                X[v] = X[bv] + 0.5 * (X[v] - X[bv])
                f[v] = energy(X[v], obj, eye)
                ev += 1
    best = sorted(range(7), key=lambda v: (f[v], order.index(v)))[0]
    return X[best], f[best]


def estimate_image(label, depth, vertex, ext, cam, factor, key, C):
    """One image.  Returns poses [C,3,4], info [C,6] and traces (hyps, per class the per-round dicts)."""
    H, W = label.shape
    fx, fy, px, py = cam
    lists = pixel_lists(label, depth, C)
    hyps = sample(label, depth, vertex, ext, cam, factor, key, lists, C)
    exhausted = sum(1 for h in hyps if h["obj"] == 0 and h["attempts"] == MAX_ATTEMPTS)
    poses = np.zeros((C, 3, 4))
    info = np.zeros((C, 6))
    rounds = {}
    for c in range(C):
        N = len(lists[c])
        ids = [h for h in range(NUM_HYP) if c > 0 and N > MIN_AREA and hyps[h]["obj"] == c]
        info[c] = (N if c else 0, len(ids), 0, -1, exhausted if c else 0, -1)
        if not ids:
            continue
        pose = {h: (hyps[h]["R"].copy(), hyps[h]["t"].copy()) for h in ids}
        L = lists[c]
        tr = []
        for r in range(ROUNDS):
            pos = subset(L, c, r, key)
            pix = (L[pos] & ~HOLE).astype(np.int64)
            eye = np.array([eye_at(depth, W, fx, fy, px, py, factor, i) for i in pix], F32).reshape(-1, 3)
            obj = np.array([mode_at(vertex, ext, c, i) for i in pix], F32).reshape(-1, 3)
            masks, near = {}, {}
            for h in ids:
                R, t = pose[h]
                d = np.linalg.norm(eye.astype(np.float64) - (obj.astype(np.float64) @ R.T + t), axis=1)
                masks[h] = np.nonzero(d < GATE)[0]
                near[h] = int(np.sum(np.abs(d - GATE) <= 1e-6 * GATE))
            cnt = {h: len(masks[h]) for h in ids}
            order = sorted(ids, key=lambda h: (-cnt[h], h))
            keep = len(ids) // 2 if len(ids) > 1 else len(ids)
            ids = order[:keep]
            tr.append(dict(taken=len(pix), hash=int(pix.sum()) & 0xFFFFFFFF, counts=cnt, near=near, best=ids[0], best_count=cnt[ids[0]],
                           subset=pix))
            last_pose = pose[ids[0]]
            for h in ids:
                inl = masks[h]
                if len(inl) < 4:
                    continue
                sel = inl if len(inl) < MAX_INL else inl[[uniform_int(words(key, ctr_fil(h, r, j))[0], len(inl)) for j in range(MAX_INL)]]
                sol = kabsch(obj[sel].astype(np.float64), eye[sel].astype(np.float64))
                if sol is not None:
                    pose[h] = sol
            if r == ROUNDS - 1:
                final_masks, final_pose0, final_eye, final_obj = masks, last_pose, eye, obj
        rounds[c] = tr
        h = ids[0]
        inl = final_masks[h]
        R, t = pose[h]
        en = -1.0
        if len(inl) > MIN_FINAL:
            if len(inl) >= MAX_INL:
                sel = [inl[uniform_int(words(key, ctr_fil(h, ROUNDS - 1, uniform_int(words(key, ctr_fil(h, ROUNDS, j))[0], MAX_INL)))[0],
                                       len(inl))] for j in range(MAX_INL)]
            else:
                sel = inl
            x0 = np.r_[rodrigues_log(R), t]
            xb, en = nelder_mead(x0, final_obj[sel], final_eye[sel])
            R, t = rodrigues_exp(xb), xb[3:]
        poses[c, :, :3], poses[c, :, 3] = R, t
        info[c, 2], info[c, 3], info[c, 5] = len(inl), en, h
    return dict(poses=poses, info=info, hyps=hyps, rounds=rounds, lists=lists)


def records(poses_tmp, ext, K, im_scale, image=0):
    """The detection records of one image (lib/fcn/test.py:1383-1399) from poses [C,3,4]: (rois [n,6], poses [n,7]) for every
    class j >= 1 with t_z > 0 in ascending order; the box projects the extent box with the pose's quaternion round trip in float32."""
    from oracle import oracle
    rois, out = [], []
    for j in range(1, poses_tmp.shape[0]):
        P = poses_tmp[j].astype(F32)
        if not P[2, 3] > 0:
            continue
        q = oracle.mat2quat(P[:, :3]).astype(F32)
        w, x, y, z = q
        s = F32(2) / (w * w + x * x + y * y + z * z)
        X, Y, Z = x * s, y * s, z * s
        R = np.array([[1 - (y * Y + z * Z), x * Y - w * Z, x * Z + w * Y], [x * Y + w * Z, 1 - (x * X + z * Z), y * Z - w * X],
                      [x * Z - w * Y, y * Z + w * X, 1 - (x * X + y * Y)]], F32)
        h = ext[j].astype(F32) * F32(0.5)
        corners = np.array([[sx * h[0], sy * h[1], sz * h[2]] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)], F32)
        cam = (corners @ R.T + P[:, 3]).astype(np.float64)
        uv = cam @ np.asarray(K, np.float64).T
        u, v = uv[:, 0] / uv[:, 2], uv[:, 1] / uv[:, 2]
        bb = np.array([u.min(), v.min(), u.max(), v.max()], F32) * F32(im_scale)
        rois.append([image, j, *bb])
        out.append([*q, *P[:, 3]])
    return np.array(rois, F32).reshape(-1, 6), np.array(out, F32).reshape(-1, 7)
