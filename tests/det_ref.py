"""NumPy restatements of the detection network's test-time stages (DESIGN.md §16), the references of tests/test_det_*.py.

Every box computation is float32 with each product and sum rounded, in the operation order of lib/utils/bbox_transform.py,
lib/nms/py_cpu_nms.py / nms_kernel.cu's devIoU and TF 1.x crop_and_resize.  Ties are ordered canonically: descending score,
then ascending flat anchor index (h, w, a).
"""
import numpy as np

F = np.float32


def decode_clip(anchors, deltas, im_h, im_w, return_scale=False):
    """bbox_transform_inv + clip_boxes on float32 [n,4] anchors and deltas.  return_scale: also the magnitude of the operands of
    each coordinate's last sum (|centre| + |half extent|), the scale at which an ulp of exp() shows up in the box."""
    a = anchors.astype(F)
    d = deltas.astype(F)
    one, half = F(1), F(0.5)
    widths = a[:, 2] - a[:, 0] + one
    heights = a[:, 3] - a[:, 1] + one
    ctr_x = a[:, 0] + half * widths
    ctr_y = a[:, 1] + half * heights
    pcx = d[:, 0] * widths + ctr_x
    pcy = d[:, 1] * heights + ctr_y
    pw = np.exp(d[:, 2]) * widths
    ph = np.exp(d[:, 3]) * heights
    boxes = np.stack([pcx - half * pw, pcy - half * ph, pcx + half * pw, pcy + half * ph], axis=1)
    xmax, ymax = F(im_w) - one, F(im_h) - one
    boxes[:, 0::2] = np.maximum(np.minimum(boxes[:, 0::2], xmax), F(0))
    boxes[:, 1::2] = np.maximum(np.minimum(boxes[:, 1::2], ymax), F(0))
    if return_scale:
        sx, sy = np.abs(pcx) + half * pw, np.abs(pcy) + half * ph
        return boxes, np.stack([sx, sy, sx, sy], axis=1)
    return boxes


def canonical_order(scores):
    """Indices by descending score, ties by ascending index."""
    s = np.asarray(scores, dtype=F).ravel()
    return np.lexsort((np.arange(s.size), -s))


def iou_row(boxes, i, rest):
    """devIoU(box i, boxes[rest]) in float32 (box i first, as nms_kernel.cu's cur_box)."""
    one = F(1)
    b = boxes.astype(F)
    xx1 = np.maximum(b[i, 0], b[rest, 0]); yy1 = np.maximum(b[i, 1], b[rest, 1])
    xx2 = np.minimum(b[i, 2], b[rest, 2]); yy2 = np.minimum(b[i, 3], b[rest, 3])
    w = np.maximum(xx2 - xx1 + one, F(0))
    h = np.maximum(yy2 - yy1 + one, F(0))
    inter = w * h
    area_i = (b[i, 2] - b[i, 0] + one) * (b[i, 3] - b[i, 1] + one)
    area_r = (b[rest, 2] - b[rest, 0] + one) * (b[rest, 3] - b[rest, 1] + one)
    return inter / (area_i + area_r - inter)


def nms_sorted(boxes, thresh, post_top_n, flipped=()):
    """Greedy NMS on boxes already in processing order: keep i unless an earlier kept box has IoU > thresh; stop at post_top_n.
    flipped: pairs (i, j), i < j, whose suppression decision is inverted (see explain_keep)."""
    n = boxes.shape[0]
    flips = {}
    for i, j in flipped:
        flips.setdefault(i, []).append(j)
    dead = np.zeros(n, dtype=bool)
    keep = []
    for i in range(n):
        if dead[i]:
            continue
        keep.append(i)
        if len(keep) == post_top_n:
            break
        rest = np.arange(i + 1, n)
        sup = iou_row(boxes, i, rest) > F(thresh)
        for j in flips.get(i, ()):
            sup[j - i - 1] = not sup[j - i - 1]
        dead[rest[sup]] = True
    return np.asarray(keep, dtype=np.int64)


def ambiguous_pairs(boxes, thresh=0.7, tol=1e-6):
    """Pairs (i, j), i < j, of boxes [n,4] whose IoU (+1 areas) in float64 lies within tol of thresh: the pairs on which two
    correct float32 evaluations of the IoU (with and without FMA contraction, or on boxes one ulp apart) may disagree."""
    b = boxes[:, :4].astype(np.float64)
    area = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    pairs = []
    for r0 in range(0, b.shape[0], 256):
        r = slice(r0, min(r0 + 256, b.shape[0]))
        w = np.maximum(np.minimum(b[r, None, 2], b[None, :, 2]) - np.maximum(b[r, None, 0], b[None, :, 0]) + 1, 0)
        h = np.maximum(np.minimum(b[r, None, 3], b[None, :, 3]) - np.maximum(b[r, None, 1], b[None, :, 1]) + 1, 0)
        inter = w * h
        iou = inter / (area[r, None] + area[None, :] - inter)
        ii, jj = np.nonzero(np.abs(iou - thresh) <= tol)
        pairs += [(int(i) + r0, int(j)) for i, j in zip(ii, jj) if i + r0 < j]
    return pairs


def explain_keep(boxes, thresh, post_top_n, want_keep, max_flips=256):
    """Show that the keep list want_keep (another NMS on the same sorted boxes) differs from nms_sorted only through ambiguous
    pairs: at each first difference, invert the decisions of the ambiguous pairs between the boxes kept so far and the box
    whose fate differs, re-run the restatement and compare the whole list again.  Returns (flipped pairs, all ambiguous pairs);
    raises AssertionError when a difference has no ambiguous pair to explain it."""
    want = np.asarray(want_keep, dtype=np.int64)
    amb = ambiguous_pairs(boxes, thresh)
    amb_by_j = {}
    for i, j in amb:
        amb_by_j.setdefault(j, set()).add(i)
    flipped = set()
    for _ in range(max_flips):
        keep = nms_sorted(boxes, thresh, post_top_n, flipped)
        if np.array_equal(keep, want):
            return sorted(flipped), amb
        m = min(keep.size, want.size)
        diff = np.nonzero(keep[:m] != want[:m])[0]
        d = int(diff[0]) if diff.size else m
        # the box whose fate differs is the earlier (in processing order) of the two boxes found at position d
        j = min(int(x[d]) for x in (keep, want) if d < x.size)
        new = {(int(i), j) for i in keep[:d] if int(i) in amb_by_j.get(j, ())} - flipped
        assert new, f"keep lists differ at position {d} (box {j}) with no IoU within 1e-6 of {thresh} to explain it"
        flipped |= new
    raise AssertionError(f"more than {max_flips} ambiguous decisions needed")


def proposal_layer(prob, deltas, anchors, im_h, im_w, pre_top_n=6000, post_top_n=300, thresh=0.7):
    """One image: prob [h,w,2A], deltas [h,w,4A] -> (rois [n,4], scores [n], sorted pre-NMS boxes [K,4], their scores [K])."""
    A = prob.shape[-1] // 2
    scores = prob[..., A:].reshape(-1).astype(F)
    boxes = decode_clip(anchors, deltas.reshape(-1, 4), im_h, im_w)
    order = canonical_order(scores)[:pre_top_n]
    pre, pre_s = boxes[order], scores[order]
    keep = nms_sorted(pre, thresh, post_top_n)
    return pre[keep], pre_s[keep], pre, pre_s


def rpn_heads(conv_rpn, w_cls, b_cls, w_box, b_box):
    """conv_rpn [..., 512] (bf16 values as float), HWIO 1x1 weights (bf16 values) -> (prob [..., 2A], deltas [..., 4A]) in float64:
    both 1x1 convolutions with ReLU, then the softmax of the pair (a, A + a)."""
    x = conv_rpn.astype(np.float64)
    s = np.maximum(x @ w_cls.reshape(512, -1).astype(np.float64) + b_cls.astype(np.float64), 0)
    d = np.maximum(x @ w_box.reshape(512, -1).astype(np.float64) + b_box.astype(np.float64), 0)
    A = s.shape[-1] // 2
    bg, fg = s[..., :A], s[..., A:]
    m = np.maximum(bg, fg)
    e0, e1 = np.exp(bg - m), np.exp(fg - m)
    return np.concatenate([e0 / (e0 + e1), e1 / (e0 + e1)], axis=-1), d


def crop_pool(feat, rois, feat_stride=16.0):
    """feat [B,H,W,C] float32 (bf16 values), rois [N,>=5] -> [N, 7*7*C] float16: crop_and_resize (TF 1.x bilinear, extrapolation 0)
    to 14 x 14 of the box / ((W-1) * stride, (H-1) * stride), then 2 x 2 max-pool, saturated to +-65504.  A batch index outside
    [0, B) crops zeros."""
    B, H, W, C = feat.shape
    N = rois.shape[0]
    out = np.zeros((N, 7, 7, C), dtype=np.float16)
    hn, wn = F(H - 1) * F(feat_stride), F(W - 1) * F(feat_stride)
    hm1, wm1, thirteen = F(H - 1), F(W - 1), F(13)
    for r in range(N):
        b = int(F(rois[r, 0]))
        x1, y1, x2, y2 = (F(rois[r, 1]) / wn, F(rois[r, 2]) / hn, F(rois[r, 3]) / wn, F(rois[r, 4]) / hn)
        hs = (y2 - y1) * hm1 / thirteen
        ws = (x2 - x1) * wm1 / thirteen
        crop = np.zeros((14, 14, C), dtype=F)
        if 0 <= b < B:
            for y in range(14):
                in_y = y1 * hm1 + F(y) * hs
                if in_y < 0 or in_y > hm1:
                    continue
                ty, by = int(np.floor(in_y)), int(np.ceil(in_y))
                yl = in_y - F(ty)
                for x in range(14):
                    in_x = x1 * wm1 + F(x) * ws
                    if in_x < 0 or in_x > wm1:
                        continue
                    lx, rx = int(np.floor(in_x)), int(np.ceil(in_x))
                    xl = in_x - F(lx)
                    tl, tr, bl, br = feat[b, ty, lx], feat[b, ty, rx], feat[b, by, lx], feat[b, by, rx]
                    top = tl + (tr - tl) * xl
                    bot = bl + (br - bl) * xl
                    crop[y, x] = top + (bot - top) * yl
        pooled = crop.reshape(7, 2, 7, 2, C).max(axis=(1, 3))
        out[r] = np.clip(pooled, -65504, 65504).astype(np.float16)
    return out.reshape(N, -1)
