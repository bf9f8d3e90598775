"""Float64 references, operand generators and launch plans for the pose-regression backward of the training step
(Trainer._pose_bwd and Trainer.update in posecnn_b200/train.py): Averagedistance (csrc/avg_distance.cu), the pose chain
l2_normalize o x weight o tanh (k_pose_chain_bwd), RoiPool's gradient (k_roi_pool_bwd) and SGD with momentum
(k_sgd_momentum).

Averagedistance, RoiPool's gradient and the momentum update are exact on dyadic operands: every product is exact and every
fp32 sum of terms on a grid g is exact in any order while the sum of their magnitudes stays below 2^24 g.  Each reference
counts that magnitude sum (the bit budget, tests/heads_ref.py) and raises BudgetExceeded at 2^24, so the kernel's result must
equal the reference bit for bit.  The pose chain goes through rsqrtf and is held to a derived fp32 error interval instead, and
the realistic Averagedistance case to a derived bound.  fmaf() emulates fp32 fused multiply-add exactly, for the momentum update
on operands that do round.

The references run in float64 on whatever device their inputs live on unless a function says otherwise.
"""
import math

import numpy as np
import torch

from tests.heads_ref import LIMIT, NUM_SMS, BudgetExceeded, check_budget, check_grid, dyadic  # noqa: F401
from tests.train_ref import quat_rot

EPS32 = 2.0 ** -24                  # unit roundoff of fp32
FP16_MAX = 65504.0


def gamma(k):
    """Higham's gamma_k = k u / (1 - k u) for fp32."""
    return k * EPS32 / (1 - k * EPS32)


# ---------------------------------------------------------------------------------------------------------------------
# 1. Averagedistance (k_average_distance): loss = sum over rows and points of max-hinge (dist - margin) / (2 N P),
#    bottom_diff = its gradient with respect to the row's (un-normalised) predicted quaternion
# ---------------------------------------------------------------------------------------------------------------------
def quat_jacobians(q):
    """[..., 4, 3, 3] d R / d (s, u, v, w) of train_ref.quat_rot (the derivative matrices of the reference's backward)."""
    s, u, v, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    m = lambda *e: torch.stack(e, -1).reshape(*q.shape[:-1], 3, 3)
    return 2 * torch.stack([m(s, -w, v, w, s, -u, -v, u, s), m(u, v, w, v, -u, -s, w, s, -u),
                            m(-v, u, s, u, v, w, -s, w, -v), m(-w, -s, u, s, -w, v, u, v, w)], -3)


def first_argmin(d):
    """Index of the first minimum over the last axis (the kernel's strict '<' scan from index 0)."""
    P = d.shape[-1]
    idx = torch.arange(P, device=d.device).expand_as(d)
    return torch.where(d == d.amin(-1, keepdim=True), idx, torch.full_like(idx, P)).amin(-1)


def row_classes(weight):
    """The first class whose weight is > 0 in each row (the kernel's class), -1 for a row without one."""
    N, D = weight.shape
    on = weight.view(N, D // 4, 4)[:, :, 0] > 0
    first = torch.where(on, torch.arange(D // 4, device=weight.device), torch.full_like(on, D // 4, dtype=torch.long)).amin(1)
    return torch.where(on.any(1), first, torch.full_like(first, -1))


def average_distance(pred, target, weight, points, symmetry, margin, chunk=8, units=None):
    """Float64 Averagedistance.  Returns dict(loss, diff [N,4C], roi_loss [N], cls [N], match [N,P] (the gt point each
    point is compared with), dist [N,P], ties (symmetric points whose minimum is attained by two distinct gt points),
    hinge_ties (points with dist == margin), sym_rows).  With units = (quaternion unit, point unit) the operands are
    checked to lie on those grids and the bit budgets of every fp32 sum in the kernel are counted (budget_*); margin must
    then lie on the grid of dist."""
    dev = pred.device
    N, D = pred.shape
    C, P = points.shape[0], points.shape[1]
    cls = row_classes(weight)
    diff = torch.zeros((N, D), dtype=torch.float64, device=dev)
    roi_loss = torch.zeros(N, dtype=torch.float64, device=dev)
    match = torch.full((N, P), -1, dtype=torch.long, device=dev)
    dist_all = torch.zeros((N, P), dtype=torch.float64, device=dev)
    out = dict(ties=0, hinge_ties=0, sym_rows=0, budget_row_grad=0.0, budget_row_loss=0.0, budget_term=0.0)
    inv_np = 1.0 / (N * P)
    if units is not None:
        uq, up = units
        ue = uq * uq * up                               # R on the grid uq^2 (2 x products of quaternion components), e = (Ru - Rg) x
        check_grid("quaternions", pred, uq)
        check_grid("targets", target, uq)
        check_grid("points", points, up)
        check_grid("margin", torch.tensor([margin]), ue * ue)
        ug = 2 * ue * up * uq                           # gs = 2 (e_j x_k q_a): the grid of a gradient term
    total_loss_units = 0.0
    rows = (cls >= 0).nonzero().flatten()
    for i0 in range(0, rows.numel(), chunk):
        r = rows[i0:i0 + chunk]
        c = cls[r]
        pq = pred.view(N, C, 4)[r, c].double()
        tq = target.view(N, C, 4)[r, c].double()
        Ru, Rg = quat_rot(pq), quat_rot(tq)
        x = points[c].double()                                           # [n,P,3]
        x1 = x @ Ru.transpose(1, 2)
        xg = x @ Rg.transpose(1, 2)                                      # gt-rotated points
        sym = symmetry[c] > 0
        j = torch.arange(P, device=dev).expand(r.numel(), P).clone()
        if bool(sym.any()):
            s = sym.nonzero().flatten()
            d2 = sum((x1[s, :, None, k] - xg[s, None, :, k]) ** 2 for k in range(3))     # [ns,P,P], exact on the grids
            j[s] = first_argmin(d2)
            # first-minimum rule observable: the minimum is attained by a gt point at another position than the first one
            mins = d2 == d2.amin(-1, keepdim=True)
            first = torch.gather(xg[s], 1, j[s, :, None].expand(-1, -1, 3))
            other = (xg[s][:, None, :, :] != first[:, :, None, :]).any(-1)           # [ns,P,P]
            out["ties"] += int((mins & other).any(-1).sum())
            out["sym_rows"] += int(s.numel())
            del d2, mins, other
        x2 = torch.gather(xg, 1, j[:, :, None].expand(-1, -1, 3))
        e = x1 - x2
        dist = (e * e).sum(-1)
        on = dist >= margin                                              # the kernel skips dist < margin
        out["hinge_ties"] += int((dist == margin).sum())
        roi_loss[r] = torch.where(on, dist - margin, torch.zeros_like(dist)).sum(1) * 0.5 * inv_np
        J = quat_jacobians(pq)                                           # [n,4,3,3]
        t = torch.einsum("npj,npk,najk->npa", e, x, J) * on[..., None]   # [n,P,4] = gs, gu, gv, gw
        diff.view(N, C, 4)[r, c] = t.sum(1) * inv_np
        match[r] = j
        dist_all[r] = dist
        if units is not None:
            check_grid("gradient terms", t, ug)
            # the nine products of one term, the per-row sums of P gradient and loss terms
            tm = torch.einsum("npj,npk,najk->npa", e.abs(), x.abs(), J.abs())
            out["budget_term"] = max(out["budget_term"], check_budget("gradient term", tm.max() / ug))
            out["budget_row_grad"] = max(out["budget_row_grad"], check_budget("row gradient", t.abs().sum(1).max() / ug))
            lu = torch.where(on, dist - margin, torch.zeros_like(dist)).abs().sum(1) / (ue * ue)
            out["budget_row_loss"] = max(out["budget_row_loss"], check_budget("row loss", lu.max()))
            total_loss_units += float(lu.sum())
    if units is not None:
        out["budget_batch_loss"] = check_budget("batch loss", total_loss_units)
    out.update(loss=roi_loss.sum(), diff=diff, roi_loss=roi_loss, cls=cls, match=match, dist=dist_all)
    return out


def ad_problem(N, C, P, gen, sym_classes=(1, 3), near_frac=0.85, none_frac=0.25, zero_frac=0.85, margin=None):
    """Dyadic Averagedistance operands: quaternion components in {-1, -1/2, 0, 1/2, 1} (not normalised), points in
    {-1/4, 0, 1/4}^3 (so gt-rotated points coincide or are equidistant from a predicted point often), a fraction zero_frac
    of them at the origin (their dist is 0: the sum of all N P loss terms must stay inside the budget), symmetry on
    sym_classes.  A fraction none_frac of the rows has no weighted class; of the others a fraction near_frac predicts a
    quaternion one step of 1/2 away from its target in one component (small distances, mostly under the margin) and the rest
    an independent one.  Some rows weight a second, later class too (the kernel must take the first).  margin defaults to
    1/64.  Returns dict(pred, target, weight, points, symmetry, margin, units)."""
    D = 4 * C
    target = dyadic((N, D), -1, 1, 0.5, gen)
    pred = dyadic((N, D), -1, 1, 0.5, gen)
    comp = torch.randint(0, 4, (N, C), generator=gen)
    step = (torch.randint(0, 2, (N, C), generator=gen) * 2 - 1).float() * 0.5
    nudged = target.view(N, C, 4).clone()
    nudged.scatter_add_(2, comp[..., None], step[..., None])
    nudged = nudged.clamp(-1, 1).view(N, D)
    kind = torch.rand(N, generator=gen)
    kind[-1] = 0.0                                                      # at least one row without a weighted class
    near =(kind >= none_frac) & (kind < none_frac + (1 - none_frac) * near_frac)
    pred = torch.where(near[:, None], nudged, pred)
    weight = torch.zeros(N, D)
    c = torch.randint(0, C, (N,), generator=gen)
    c[: 2 * len(sym_classes)] = torch.tensor(list(sym_classes) * 2)     # every symmetric class is present
    for n in range(N):
        if kind[n] < none_frac:
            continue
        weight[n, 4 * c[n]:4 * c[n] + 4] = 1.0
        if n % 5 == 0 and c[n] + 1 < C:
            weight[n, 4 * (C - 1):4 * C] = 1.0                           # a second, later weighted class
    points = dyadic((C, P, 3), -0.25, 0.25, 0.25, gen)
    points[torch.rand(C, P, generator=gen) < zero_frac] = 0.0            # dist 0 under any rotation: keeps the batch budget
    symmetry = torch.zeros(C)
    symmetry[list(sym_classes)] = 1.0
    return dict(pred=pred, target=target, weight=weight, points=points, symmetry=symmetry,
                margin=1.0 / 64 if margin is None else margin, units=(0.5, 0.25))


def ad_plan(N, P):
    """One CTA of 256 threads per row; each thread runs ceil(P / 256) points serially, then a 256-leaf tree; the last CTA
    to finish reduces the N row losses."""
    return dict(grid=N, threads=256, points_per_thread=math.ceil(P / 256), batch_items_per_thread=math.ceil(N / 256))


def ad_bound(pred, target, weight, points, symmetry, margin, ref, chunk=8):
    """Derived error bounds of the fp32 kernel against the float64 reference on arbitrary (non-dyadic) operands.
    A point's fp32 dist, e and gradient terms are formed in at most K_TERM rounding steps; its sum runs over
    ceil(P/256) serial additions and a tree of 8 levels; the batch loss over ceil(N/256) + 8 more.  Every |x1_j| + |x2_j| is
    bounded by A = |q_pred|^2 sum|x| + |q_gt|^2 max_i sum|x_i| (any gt point a symmetric search may choose).  A point is
    ambiguous when its float64 dist lies within the dist error of the margin, or when another gt point's distance lies
    within twice that error of the minimum: its whole possible contribution (twice the magnitude bound) is added to the
    bound.  Returns dict(grad [N,4C] bound, loss bound, ambiguous count)."""
    K_TERM = 24
    dev = pred.device
    N, D = pred.shape
    C, P = points.shape[0], points.shape[1]
    inv_np = 1.0 / (N * P)
    depth = math.ceil(P / 256) + 8
    g_row = gamma(K_TERM + depth + 1)                    # + 1: inv_np is rounded to fp32
    cls = ref["cls"]
    bound = torch.zeros((N, D), dtype=torch.float64, device=dev)
    loss_bound = 0.0
    ambiguous = 0
    rows = (cls >= 0).nonzero().flatten()
    for i0 in range(0, rows.numel(), chunk):
        r = rows[i0:i0 + chunk]
        c = cls[r]
        pq = pred.view(N, C, 4)[r, c].double()
        tq = target.view(N, C, 4)[r, c].double()
        x = points[c].double()
        xs = x.abs().sum(-1)                                                          # [n,P]
        A = (pq * pq).sum(-1)[:, None] * xs + (tq * tq).sum(-1)[:, None] * xs.amax(1, keepdim=True)
        derr = gamma(K_TERM) * 3 * A * A                                              # |dist error|
        dist = ref["dist"][r]
        amb = (dist - margin).abs() <= derr
        sym = symmetry[c] > 0
        if bool(sym.any()):
            s = sym.nonzero().flatten()
            Ru, Rg = quat_rot(pq[s]), quat_rot(tq[s])
            x1, xg = x[s] @ Ru.transpose(1, 2), x[s] @ Rg.transpose(1, 2)
            d2 = sum((x1[:, :, None, k] - xg[:, None, :, k]) ** 2 for k in range(3))
            dmin = d2.amin(-1, keepdim=True)
            close = (d2 - dmin <= 2 * derr[s][:, :, None]).sum(-1) > 1
            amb[s] |= close
            del d2
        J = quat_jacobians(pq).abs()
        G = torch.einsum("np,npk,najk->npa", A, x.abs(), J)                           # magnitude bound of a point's 4 terms
        Lm = 0.5 * ((dist - margin).abs() + derr)                                     # of its loss term
        ambiguous += int(amb.sum())
        wide = amb[..., None].double()
        bound.view(N, C, 4)[r, c] = (g_row * G.sum(1) + 2 * (G * wide).sum(1)) * inv_np
        loss_bound += float(((g_row + gamma(math.ceil(N / 256) + 8)) * Lm.sum() + 2 * (Lm * amb).sum()) * inv_np)
    return dict(grad=bound, loss=loss_bound, ambiguous=ambiguous)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the pose chain (k_pose_chain_bwd): d pre = d/d pre of l2_normalize(tanh(pre) * w) applied to upstream * g
# ---------------------------------------------------------------------------------------------------------------------
CLAMP = 1e-12


def pose_chain(g, tanhv, wgt, upstream):
    """Float64 d pre [N,D] and a per-element bound of the fp32 kernel's error (before its fp16 rounding).
    u = t w, su = sum u^2 (clamped at fp32(1e-12)), inv = su^-1/2, du = (g - u inv^2 (u.g)) inv, d = du w (1 - t^2).
    The kernel's su and u.g are fp32 sums of D / 32 serial fmaf's and a 5-level butterfly, inv = rsqrtf (2 ulp), and du and d
    take 7 more roundings.  The bound is first-order in those errors, doubled.  The clamp decision is taken in float64; the
    operands keep su far from 1e-12."""
    g, t, w = g.double(), tanhv.double(), wgt.double()
    gg = upstream * g
    u = t * w
    su = (u * u).sum(1, keepdim=True)
    clamped = su < float(np.float32(CLAMP))
    inv = torch.where(clamped, torch.full_like(su, float(np.float32(CLAMP)) ** -0.5), su.clamp(min=float(np.float32(CLAMP))).rsqrt())
    ug = torch.where(torch.isfinite(gg), u * gg, torch.zeros_like(gg)).sum(1, keepdim=True)   # non-finite g only in clamped rows
    du = torch.where(clamped, gg * inv, (gg - u * inv * inv * ug) * inv)
    d = du * w * (1 - t * t)
    k = math.ceil(g.shape[1] / 32) + 5
    d_inv = 2 * 2.0 ** -23 + gamma(k) / 2                                   # relative error of inv
    e_ug = gamma(k) * torch.where(torch.isfinite(gg), (u * gg).abs(), torch.zeros_like(gg)).sum(1, keepdim=True)
    proj = u.abs() * inv ** 3 * ug.abs()
    err_du = torch.where(clamped, (gg * inv).abs() * (d_inv + EPS32),
                         (gg * inv).abs() * (d_inv + 2 * EPS32) + proj * (3 * d_inv + 5 * EPS32) + u.abs() * inv ** 3 * e_ug)
    err = 2 * ((w * (1 - t * t)).abs() * err_du + du.abs() * w.abs() * EPS32 * (t * t + (1 - t * t).abs()) + 3 * EPS32 * d.abs())
    return d, err, clamped.flatten()


def f16_sat(x):
    """fp16 of the saturated value: +-inf and finite overflow to +-65504, NaN stays NaN (then round to nearest even)."""
    x = x.double()
    return torch.where(torch.isnan(x), x, x.clamp(-FP16_MAX, FP16_MAX)).to(torch.float16)


def pose_chain_problem(N, C, gen, ld=None):
    """Operands of the step's pose chain: one-hot class weight blocks (every fifth row dense weights in [1/2, 3/2]), tanh of
    N(0, 1) pre-activations, g ~ N(0, 1e-4) (the size of an Averagedistance gradient).  Row 0 (if N > 2) has all-zero
    weights, row 1 tanh values of 1e-9 (sum u^2 < 1e-12): both are clamped rows."""
    D = 4 * C
    t = torch.tanh(torch.randn(N, D, generator=gen))
    w = torch.zeros(N, D)
    c = torch.randint(0, C, (N,), generator=gen)
    w.view(N, C, 4)[torch.arange(N), c] = 1.0
    dense = torch.arange(N) % 5 == 4
    w[dense] = 0.5 + torch.rand(int(dense.sum()), D, generator=gen)
    g = torch.randn(N, D, generator=gen) * 1e-4
    if N > 2:
        w[0] = 0.0
        t[1] = 1e-9 * torch.sign(t[1])
    return dict(g=g, tanh=t, w=w, D=D, ld=ld or (D + 127) // 128 * 128)


def pose_chain_plan(N, D, ld):
    """One warp per row, 8 rows per CTA of 256 threads; a lane runs ceil(D / 32) columns of the sums and ceil(ld / 32) of the
    output."""
    return dict(grid=math.ceil(N / 8), rows_per_cta=8, last_cta_rows=N - 8 * (math.ceil(N / 8) - 1), cols_per_lane=math.ceil(D / 32),
                out_per_lane=math.ceil(ld / 32))


# ---------------------------------------------------------------------------------------------------------------------
# 4. RoiPool's gradient (k_roi_pool_bwd): a scatter through the forward's argmax, with the reference's three acceptance tests
# ---------------------------------------------------------------------------------------------------------------------
def roundf(x):
    """C roundf (half away from zero) of float32 values, as int64."""
    x = x.double()
    return (torch.sign(x) * torch.floor(x.abs() + 0.5)).long()


def roi_geometry(rois, scale, ph_n=7, pw_n=7):
    """Per row: batch index, the rounded corners at `scale` (fp32 product, roundf) and the fp32 bin sizes."""
    r = rois.float()
    b = torch.trunc(r[:, 0]).long()
    sc = torch.tensor(scale, dtype=torch.float32)
    rsw, rsh, rew, reh = (roundf(r[:, k] * sc) for k in (2, 3, 4, 5))
    rw = (rew - rsw + 1).clamp(min=1)
    rh = (reh - rsh + 1).clamp(min=1)
    bh = rh.float() / torch.tensor(float(ph_n), dtype=torch.float32)
    bw = rw.float() / torch.tensor(float(pw_n), dtype=torch.float32)
    return dict(b=b, rsw=rsw, rsh=rsh, rew=rew, reh=reh, bh=bh, bw=bw)


def roi_accepts(geo, argmax, H, W, Cc, ph_n=7, pw_n=7):
    """[N,ph,pw,C] bool: the (bin, element) pair the argmax names is accepted by the reference's gather
    (roi_pooling_op_gpu.cu.cc:153-211): the element lies inside the un-clipped roi, the bin lies in the element's feasible
    bin range (fp32 divisions, floor / ceil, clamped to the grid) and the argmax names it (a >= 0)."""
    N = argmax.shape[0]
    a = argmax.long()
    pix = a.clamp(min=0) // Cc
    h, w = pix // W, pix % W
    G = {k: v.view(N, 1, 1, 1) for k, v in geo.items()}
    inside = (w >= G["rsw"]) & (w <= G["rew"]) & (h >= G["rsh"]) & (h <= G["reh"])
    f = lambda num, den: num.float() / den                       # fp32 division, like __fdiv_rn
    phs = torch.floor(f(h - G["rsh"], G["bh"])).long().clamp(0, ph_n)
    phe = torch.ceil(f(h - G["rsh"] + 1, G["bh"])).long().clamp(0, ph_n)
    pws = torch.floor(f(w - G["rsw"], G["bw"])).long().clamp(0, pw_n)
    pwe = torch.ceil(f(w - G["rsw"] + 1, G["bw"])).long().clamp(0, pw_n)
    ph = torch.arange(ph_n).view(1, ph_n, 1, 1)
    pw = torch.arange(pw_n).view(1, 1, pw_n, 1)
    return (a >= 0) & inside & (ph >= phs) & (ph < phe) & (pw >= pws) & (pw < pwe)


def roi_pool_grad(shape, rois, argmax, dpool, scale, unit):
    """Float64 RoiPoolGrad on the CPU: bottom_diff [B,H,W,C].  Rows whose batch index lies outside [0, B) add nothing.
    dpool must lie on the grid `unit`; the budget is the largest per-element sum of |contributions| in units.  Returns
    (grad, budget, accepted count)."""
    B, H, W, Cc = shape
    rois, argmax, dpool = rois.cpu(), argmax.cpu(), dpool.cpu()
    check_grid("dpool", dpool, unit)
    geo = roi_geometry(rois, scale, argmax.shape[1], argmax.shape[2])
    ok = roi_accepts(geo, argmax, H, W, Cc, argmax.shape[1], argmax.shape[2])
    ok &= ((geo["b"] >= 0) & (geo["b"] < B)).view(-1, 1, 1, 1)
    flat = geo["b"].view(-1, 1, 1, 1).clamp(0, B - 1) * (H * W * Cc) + argmax.long().clamp(min=0)
    idx = flat[ok]
    out = torch.zeros(B * H * W * Cc, dtype=torch.float64).index_add_(0, idx, dpool.double()[ok])
    mag = torch.zeros(B * H * W * Cc, dtype=torch.float64).index_add_(0, idx, dpool.double()[ok].abs())
    return out.view(B, H, W, Cc), check_budget("roi_pool_grad", mag.max() / unit), int(ok.sum())


def train_rois(gen, img_h=480, img_w=640, boxes=115, B=2):
    """RoiPool rows [b, cls, x1, y1, x2, y2, score] the way Hough voting's train mode emits them: 9 jittered rows per box
    (the box, then 8 copies with corners moved by up to 1/8 of its size), heavily overlapping.  Corners are multiples of
    1/2 pixel, so many land on .5 after the 1/8 and 1/16 scalings (roundf rounds those away from zero).  Adds boxes
    crossing every border, a whole-image box, a malformed box (x2 < x1) and rows with batch index -1 and B (what a
    batch_offset produces for another rank's images)."""
    rows = []
    for k in range(boxes):
        w = 32 + float(torch.randint(0, 288, (1,), generator=gen))
        h = 32 + float(torch.randint(0, 224, (1,), generator=gen))
        x1 = float(torch.randint(-24, img_w - 8, (1,), generator=gen))
        y1 = float(torch.randint(-24, img_h - 8, (1,), generator=gen))
        b, c = k % B, 1 + k % 5
        for j in range(9):
            jit = torch.zeros(4) if j == 0 else (torch.rand(4, generator=gen) - 0.5) * torch.tensor([w, h, w, h]) / 4
            x = torch.round((torch.tensor([x1, y1, x1 + w, y1 + h]) + jit) * 2) / 2     # half-pixel grid
            if j % 3 == 1:
                x = torch.round(x / 16) * 16 + 8                         # k + 1/2 at scale 1/16
            elif j % 3 == 2:
                x = torch.round(x / 8) * 8 + 4                           # k + 1/2 at scale 1/8
            rows.append([b, c, *x.tolist(), 1.0])
    rows += [[0, 1, -40, -30, 100, 90, 1.0], [1, 2, 560, 400, 700, 520, 1.0], [0, 3, -8, 200, 120, 488, 1.0],
             [0, 4, -8, -4, 200, 180, 1.0], [1, 5, -24, -12, 40, 36, 1.0],
             [1, 1, 0, 0, img_w - 1, img_h - 1, 1.0], [0, 2, 300, 100, 200, 200, 1.0], [1, 4, 260, 300, 120, 200, 1.0],
             [-1, 1, 100, 100, 300, 300, 1.0], [B, 2, 50, 60, 250, 260, 1.0], [B + 1, 3, 0, 0, 639, 479, 1.0]]
    return torch.tensor(rows, dtype=torch.float32)


def roi_bwd_plan(N, Cc, bins=49):
    """k_roi_pool_bwd<4>: one thread per (row, bin, 4 channels), grid capped at 16 waves of 132 CTAs."""
    total = N * bins * (Cc // 4)
    grid = min(math.ceil(total / 256), NUM_SMS * 16)
    return dict(grid=grid, items=total, items_per_thread=math.ceil(total / (grid * 256)))


# ---------------------------------------------------------------------------------------------------------------------
# 5. SGD with momentum (k_sgd_momentum): a = fmaf(mu, accum, fmaf(wd, w, gscale * g)); w = fmaf(-lr, a, w)
# ---------------------------------------------------------------------------------------------------------------------
def _round32_directed(s64, r):
    """The fp32 neighbours (lo, hi) of float64 values s64 around their round-to-nearest r."""
    r64 = r.double()
    up = torch.nextafter(r, torch.full_like(r, math.inf))
    dn = torch.nextafter(r, torch.full_like(r, -math.inf))
    lo = torch.where(r64 <= s64, r, dn)
    hi = torch.where(r64 >= s64, r, up)
    return lo, hi


def fmaf(a, b, c):
    """Exact fp32 fused multiply-add of float32 tensors (a * b + c rounded once to nearest even).  The product is exact in
    float64; TwoSum gives the float64 sum and its residual; where the float64 sum is an fp32 midpoint, the residual's sign
    decides the direction (elsewhere float64 rounding cannot cross a midpoint).  Non-finite values follow IEEE."""
    p = a.double() * b.double()
    c64 = c.double()
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    r = s.float()
    lo, hi = _round32_directed(s, r)
    mid = torch.isfinite(s) & (lo != hi) & ((lo.double() + hi.double()) * 0.5 == s)
    err = torch.where(torch.isfinite(err), err, torch.zeros_like(err))
    return torch.where(mid & (err > 0), hi, torch.where(mid & (err < 0), lo, r))


def sgd_fp32(w, accum, g, lr, mu, wd, gscale):
    """k_sgd_momentum emulated bit for bit on float32 tensors (hyperparameters rounded to fp32 as the C ABI passes them).
    Returns (w', accum')."""
    f = lambda x: torch.full_like(w, x)                 # rounded to fp32
    gs = (f(gscale) * g) if gscale != 1.0 else g
    a = fmaf(f(mu), accum, fmaf(f(wd), w, gs))
    return fmaf(-f(lr), a, w), a


def sgd_fp32_chunked(w, accum, g, lr, mu, wd, gscale, chunk=1 << 24):
    """sgd_fp32 on the CPU in chunks (bounded float64 temporaries)."""
    wo, ao = torch.empty_like(w), torch.empty_like(accum)
    for i in range(0, w.numel(), chunk):
        wo[i:i + chunk], ao[i:i + chunk] = sgd_fp32(w[i:i + chunk], accum[i:i + chunk], g[i:i + chunk], lr, mu, wd, gscale)
    return wo, ao


def sgd_f64(w, accum, g, lr, mu, wd, gscale):
    """The MomentumOptimizer step in float64, unrounded: accum' = mu accum + (wd w + gscale g), w' = w - lr accum'."""
    a = mu * accum.double() + (wd * w.double() + gscale * g.double())
    return w.double() - lr * a, a


SGD_DYADIC = dict(lr=2.0 ** -7, mu=7.0 / 8.0, wd=2.0 ** -10, gscale=2.0 ** -2)


def tie_values(w, kind):
    """The value nearest to w whose 16-bit rounding is a tie (bf16: low 16 bits 0x8000; fp16: low 13 bits 0x1000), in
    [1/2, 1) with w's sign (w must lie in [1/2, 1) in magnitude)."""
    q = 2.0 ** -9 if kind == "bf16" else 2.0 ** -12              # grid of a tie value in [1/2, 1): odd multiples of q
    k = torch.floor(w.double().abs() / (2 * q))
    return torch.sign(w.double()) * ((2 * k + 1) * q).clamp(0.5 + q, 1 - q)


def sgd_step_operands(w, accum, gen, kind, tie_frac=0.25):
    """A gradient g for the state (w, accum) under SGD_DYADIC such that every fmaf of the step is exact: a target momentum
    a on the grid 2^-4 (2^-5 for the fp16 ties) is drawn in [-2, 2] (or chosen so that w - lr a is a rounding tie of the
    16-bit copy for a fraction tie_frac of the elements in [1/2, 1)), and g = (a - mu accum - wd w) / gscale.  Raises
    BudgetExceeded if g, or any intermediate of the step, is not exactly an fp32 value."""
    H = SGD_DYADIC
    n = w.numel()
    a = dyadic((n,), -2, 2, 2.0 ** -4, gen).double()
    big = (w.abs() >= 0.5) & (w.abs() < 1)
    tie = big & (torch.rand(n, generator=gen) < tie_frac / max(float(big.double().mean()), 1e-9))
    a = torch.where(tie, (w.double() - tie_values(w, kind)) / H["lr"], a)
    g = (a - H["mu"] * accum.double() - H["wd"] * w.double()) / H["gscale"]
    inner = H["wd"] * w.double() + H["gscale"] * g
    for what, x in (("g", g), ("wd w + gscale g", inner), ("accum", a), ("w", w.double() - H["lr"] * a)):
        if not bool((x.float().double() == x).all()):
            raise BudgetExceeded(f"sgd: {what} is not exactly an fp32 value")
    return g.float(), tie


def ew_plan(n):
    """Grid-stride element-wise kernels (ew_blocks in csrc/train_bwd.cu): min(ceil(n / 256), 8 x 132) CTAs of 256 threads."""
    grid = min(math.ceil(n / 256), NUM_SMS * 8)
    return dict(grid=grid, items_per_thread=math.ceil(n / (grid * 256)), ragged=n % (grid * 256) != 0)
