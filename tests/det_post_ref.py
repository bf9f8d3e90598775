"""NumPy restatement of the detection network's test-loop records (DESIGN.md §16), the reference of tests/test_det_post_*.py and
of posecnn_b200/det_records.py (csrc/det.cu: k_det_records).

    denormalise    fcn/test.py:1731-1734   bbox_pred *= stds (float64), += means (0), stored back into the float32 array
    class_boxes    fcn/test.py:1736-1743   bbox_transform_inv + clip_boxes (utils/bbox_transform.py), float32
    select         fcn/test.py:1593-1604   per class j >= 1: the top cls_prob[:, j] > 0.02 (nms(...)[0] is the top score);
                                           exact ties go to the lowest row (the reference's argsort()[::-1] leaves them open)
    objective      fcn/test.py:1668-1691   distance_objective in the device's operation order: fp32 camera coordinates
                                           ((r0 px + r1 py) + r2 pz) + t, elementwise (numpy's float32 ops are correctly rounded,
                                           never fused), then K's row products, the division and the extents in float64
    nelder_mead    scipy 1.18.1 _minimize_neldermead at N = 1 (x0 = 0.5, defaults), with every comparison recorded
    translation    fcn/test.py:1639-1664   compute_translations of one record

Every comparison of the search is recorded with its margin (the distance between the compared values) and the objective's
fp32 sensitivity at the values compared (`sensitivity`).  `replay` runs the search on another correct evaluation's objective
values (the reference's BLAS sgemm sums RT @ x3d in its own order, with FMA) and lists the decisions the two take
differently, each of which must lie within that sensitivity.
"""
import math

import numpy as np

from tests.eval_ref import quat2mat

F = np.float32
STDS = np.array([0.1, 0.1, 0.2, 0.2])                   # config.py:199 TRAIN.BBOX_NORMALIZE_STDS
MEANS = np.array([0.0, 0.0, 0.0, 0.0])                  # config.py:197
THRESH = F(0.02)                                        # test.py:1592
MAXFUN = 200                                            # N * 200 (maxiter = maxfun)
XATOL = FATOL = 1e-4
U = 2.0 ** -24                                          # fp32 unit roundoff
SENS_ULPS = 8                                           # roundings per camera coordinate the other evaluation may differ by


def denormalise(bbox_pred):
    """test.py:1731-1734 on float32 [n,4C]: each delta becomes f32(f64(d) * std) (+ 0.0)."""
    d = np.array(bbox_pred, dtype=F)
    C = d.shape[1] // 4
    d *= np.tile(STDS, C)
    d += np.tile(MEANS, C)
    return d


def class_boxes(rois, deltas, im_h, im_w):
    """bbox_transform_inv(rois[:, 1:5], deltas) + clip_boxes(.., (im_h, im_w)) on float32 [n,5] / [n,4C] -> [n,4C]."""
    b = np.asarray(rois, F)[:, 1:5]
    d = np.asarray(deltas, F)
    one, half = F(1), F(0.5)
    widths = (b[:, 2] - b[:, 0] + one)[:, None]
    heights = (b[:, 3] - b[:, 1] + one)[:, None]
    ctr_x = b[:, 0:1] + half * widths
    ctr_y = b[:, 1:2] + half * heights
    pcx = d[:, 0::4] * widths + ctr_x
    pcy = d[:, 1::4] * heights + ctr_y
    pw = np.exp(d[:, 2::4]) * widths
    ph = np.exp(d[:, 3::4]) * heights
    out = np.zeros(d.shape, F)
    out[:, 0::4], out[:, 1::4] = pcx - half * pw, pcy - half * ph
    out[:, 2::4], out[:, 3::4] = pcx + half * pw, pcy + half * ph
    out[:, 0::2] = np.maximum(np.minimum(out[:, 0::2], im_w - 1), 0)
    out[:, 1::2] = np.maximum(np.minimum(out[:, 1::2], im_h - 1), 0)
    return out


def select(scores, n):
    """[(j, row)] for j = 1..C-1 with a score > 0.02 among rows < n: the top score, ties to the lowest row (np.argmax)."""
    out = []
    s = np.asarray(scores, F)[:n]
    for j in range(1, s.shape[1]):
        inds = np.where(s[:, j] > THRESH)[0]
        if inds.size:
            out.append((j, int(inds[np.argmax(s[inds, j])])))
    return out


def objective(z, R, rx, ry, pts, K, width, height, want_sens=False):
    """distance_objective(z) in the device's operation order.  R [3,3] f32, pts [P,3] f32, K [3,3] f64, width / height f32.
    want_sens: also the fp32 sensitivity (see `sensitivity`)."""
    t = (F(rx * z), F(ry * z), F(z))
    px, py, pz = pts[:, 0], pts[:, 1], pts[:, 2]
    cam = [((R[r, 0] * px + R[r, 1] * py) + R[r, 2] * pz) + t[r] for r in range(3)]
    c = [v.astype(np.float64) for v in cam]
    q = [(K[r, 0] * c[0] + K[r, 1] * c[1]) + K[r, 2] * c[2] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = q[0] / q[2], q[1] / q[2]
        w = np.max(u) - np.min(u)
        h = np.max(v) - np.min(v)
        dw, dh = w - np.float64(width), h - np.float64(height)
        f = dw * dw + dh * dh
    if not want_sens:
        return float(f)
    return float(f), sensitivity(R, t, pts, K, c, float(dw), float(dh))


def sensitivity(R, t, pts, K, c, dw, dh):
    """How far another correct fp32 evaluation of the camera coordinates can move f: each coordinate X = r0 px + r1 py + r2 pz
    + t may differ by SENS_ULPS roundings of its terms' magnitude S_X (another summation order, or FMA); through u = fx X / Z
    + cx that moves a projected coordinate by fx (dX / |Z| + |X| dZ / Z^2), an extent by twice the largest such move D, and
    f = dw^2 + dh^2 by 2 (|dw| + |dh|) 2D + 8 D^2."""
    a = np.abs(pts.astype(np.float64))
    S = [np.abs(R[r].astype(np.float64)) @ a.T + abs(float(t[r])) for r in range(3)]
    e = [SENS_ULPS * U * s for s in S]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        Z = np.abs(c[2])
        du = abs(K[0, 0]) * (e[0] / Z + np.abs(c[0]) * e[2] / (Z * Z))
        dv = abs(K[1, 1]) * (e[1] / Z + np.abs(c[1]) * e[2] / (Z * Z))
        D = float(max(np.max(du), np.max(dv)))
        s = 4 * (abs(dw) + abs(dh)) * D + 8 * D * D
    return s if math.isfinite(s) else math.inf


class Value(float):
    """An objective value that drives the search, with the restatement's own value of the same point (alt) and its fp32
    sensitivity (sens)."""

    def __new__(cls, f, alt=None, sens=0.0):
        v = super().__new__(cls, f)
        v.alt, v.sens = (float(f) if alt is None else float(alt)), float(sens)
        return v


def _lt(a, b):
    return a < b


def _le(a, b):
    return a <= b


def _sorts_before(b, a):
    """np.argsort of (a, b): stable, NaN last, so b comes first when b < a or a alone is NaN."""
    return b < a or (a != a and b == b)


def _converged(a, b):
    return abs(a - b) <= FATOL


class Search:
    """One Nelder-Mead run with its decision record.  fn(z) -> Value.  xs / fs: the evaluated points and values in order;
    decisions: (kind, taken, taken on the alt values, margin of the alt values, tolerance, evaluations done before it)."""

    def __init__(self, fn):
        self.fn = fn
        self.xs, self.fs, self.decisions = [], [], []

    def call(self, x):
        if len(self.xs) >= MAXFUN:
            raise StopIteration                          # _MaxFuncCallError
        f = self.fn(x)
        self.xs.append(x), self.fs.append(f)
        return f

    def decide(self, kind, op, a, b):
        taken, alt = op(a, b), op(a.alt, b.alt)
        d = abs(a.alt - b.alt)
        margin = abs(d - FATOL) if op is _converged else d
        self.decisions.append((kind, taken, alt, margin if margin == margin else math.inf, a.sens + b.sens, len(self.xs)))
        return taken

    def run(self):
        s0, s1 = 0.5, (1 + 0.05) * 0.5
        f0, f1 = self.call(s0), self.call(s1)
        if self.decide("sort", _sorts_before, f1, f0):
            s0, s1, f0, f1 = s1, s0, f1, f0
        it = 1
        while len(self.xs) < MAXFUN and it < MAXFUN:
            if abs(s1 - s0) <= XATOL and self.decide("fatol", _converged, f0, f1):
                break
            try:
                xbar = s0
                xr = 2.0 * xbar - 1.0 * s1
                fxr = self.call(xr)
                if self.decide("reflect", _lt, fxr, f0):
                    xe = 3.0 * xbar - 2.0 * s1
                    fxe = self.call(xe)
                    if self.decide("expand", _lt, fxe, fxr):
                        s1, f1 = xe, fxe
                    else:
                        s1, f1 = xr, fxr
                else:                                    # N = 1: fsim[-2] is fsim[0], so `fxr < fsim[-2]` cannot hold here
                    shrink = False
                    if self.decide("outside", _lt, fxr, f1):
                        xc = 1.5 * xbar - 0.5 * s1
                        fxc = self.call(xc)
                        if self.decide("contract", _le, fxc, fxr):
                            s1, f1 = xc, fxc
                        else:
                            shrink = True
                    else:
                        xcc = 0.5 * xbar + 0.5 * s1
                        fxcc = self.call(xcc)
                        if self.decide("inside", _lt, fxcc, f1):
                            s1, f1 = xcc, fxcc
                        else:
                            shrink = True
                    if shrink:
                        s1 = s0 + 0.5 * (s1 - s0)
                        f1 = self.call(s1)
                it += 1
            except StopIteration:
                pass
            if self.decide("sort", _sorts_before, f1, f0):
                s0, s1, f0, f1 = s1, s0, f1, f0
        self.z, self.nit, self.nfev = s0, it, len(self.xs)
        return self


def fit_inputs(box, q, pts, K):
    """compute_translations' per-record quantities: (R f32, rx, ry, width, height) of box (x1, y1, x2, y2) f32."""
    x1, y1, x2, y2 = (F(v) for v in box)
    x, y = (x1 + x2) / F(2), (y1 + y2) / F(2)
    rx = (np.float64(x) - K[0, 2]) / K[0, 0]
    ry = (np.float64(y) - K[1, 2]) / K[1, 1]
    return quat2mat(q).astype(F), float(rx), float(ry), x2 - x1, y2 - y1


def translation(box, q, pts, K):
    """compute_translations of one record: box (x1, y1, x2, y2) f32, q [4] f32, pts [P,3] f32, K [3,3] f64 -> (t [3] f32, Search)."""
    R, rx, ry, width, height = fit_inputs(box, q, pts, K)
    pts = np.asarray(pts, F)
    s = Search(lambda z: Value(objective(z, R, rx, ry, pts, K, width, height))).run()
    return np.array([rx * s.z, ry * s.z, s.z], F), s


def records(cls_prob, bbox_pred, poses_tanh, rois, num_rois, im_hw, meta, points):
    """The whole stage for B images of N rows (the layout of det_records.detection_records) -> dets [B*(C-1),7], poses
    [B*(C-1),7], num_dets [B], trace [B*(C-1),2], boxes [B*N,4C]."""
    cls_prob, rois = np.asarray(cls_prob, F), np.asarray(rois, F)
    B = len(num_rois)
    rows, C = cls_prob.shape
    N = rows // B
    boxes = class_boxes(rois, denormalise(bbox_pred), *im_hw)
    dets = np.zeros((B * (C - 1), 7), F)
    poses = np.zeros((B * (C - 1), 7), F)
    trace = np.zeros((B * (C - 1), 2), np.int32)
    num = np.zeros(B, np.int32)
    dets[:, 0] = np.repeat(np.arange(B), C - 1)
    for b in range(B):
        K = np.asarray(meta[b][:9], F).astype(np.float64).reshape(3, 3)
        for j, r in select(cls_prob[b * N:(b + 1) * N], int(num_rois[b])):
            row, slot = b * N + r, b * (C - 1) + j - 1
            box = boxes[row, 4 * j:4 * j + 4]
            q = np.asarray(poses_tanh[row, 4 * j:4 * j + 4], F)
            t, s = translation(box, q, points[j], K)
            dets[slot] = [b, j, *box, cls_prob[row, j]]
            poses[slot] = [*q, *t]
            trace[slot] = (s.nit, s.nfev)
            num[b] += 1
    return dets, poses, num, trace, boxes


def replay(box, q, pts, K, want_xs, want_fs):
    """Run the restated search on another evaluation's objective values (want_fs at the points want_xs, e.g. the reference's),
    with the restatement's own values alongside.  Returns the Search (its xs must be want_xs if the two searches are the same
    algorithm) and the decisions the two sets of values take differently [(kind, margin, tolerance)]: each must lie within
    the objective's fp32 sensitivity for the difference to be explained by the objective's rounding alone."""
    R, rx, ry, width, height = fit_inputs(box, q, pts, K)
    pts = np.asarray(pts, F)
    table = dict(zip(map(float, want_xs), map(float, want_fs)))

    def fn(z):
        assert z in table, f"the replayed search evaluates z = {z!r}, which the other search never did"
        mine, sens = objective(z, R, rx, ry, pts, K, width, height, want_sens=True)
        return Value(table[z], mine, sens)
    s = Search(fn).run()
    return s, [(d[0], d[3], d[4]) for d in s.decisions if d[1] != d[2]]
