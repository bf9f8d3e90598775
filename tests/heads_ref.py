"""Dyadic operands, float64 references and launch plans for the FCN-head kernels of the training step and of inference
(csrc/heads.cu, csrc/train_bwd.cu, the classification loss of csrc/train_targets.cu).

The heads are linear or piecewise linear in their inputs, and their fixed weights are dyadic: the bilinear x8 taps are
multiples of 1/16, the x2 taps are 1/4 and 3/4.  With operands on a dyadic grid every product is exact, and a sum of terms
that are all multiples of a unit g is exact in fp32 in ANY order as long as the sum of their magnitudes stays below 2^24 g
(every partial sum is then an integer multiple of g below 2^24 g).  Each reference here computes, next to its result, that
magnitude sum in units of its granularity (the "bit budget") and raises BudgetExceeded when it reaches 2^24.  Exactness is
then a checked condition, and the kernel's output must equal the reference rounded once (bf16 round-to-nearest-even, or
fp32), bit for bit.

Tensors are NHWC.  The references run in float64 on whatever device their inputs live on.
"""
import math

import numpy as np
import torch

from tests.util import int_operands

LIMIT = 1 << 24
NUM_SMS = 132                   # kNumSMs (csrc/common.cuh): the block caps of the element-wise and head kernels


class BudgetExceeded(AssertionError):
    """An fp32 sum of the terms could round: the operand range is too wide for an exact comparison."""


def check_budget(what, units):
    units = float(units)
    if not units < LIMIT:
        raise BudgetExceeded(f"{what}: {units:.0f} units of granularity >= 2^24, an fp32 sum of these terms may round")
    return units


def check_grid(what, t, unit):
    """Every element of t is an integer multiple of `unit` (the granularity a budget is counted in)."""
    q = t.double() / unit
    assert bool((q == q.round()).all()), f"{what}: not on the grid of {unit}"


def dyadic(shape, lo, hi, unit, gen):
    """Seeded float32 CPU tensor of multiples of `unit` drawn uniformly from [lo, hi]."""
    return int_operands(shape, round(lo / unit), round(hi / unit), gen) * unit


def bilinear_taps(k):
    """make_deconv_filter's 1-D factor (deconv_w, csrc/heads_common.cuh): f = ceil(k/2), c = (2f - 1 - f%2) / (2f)."""
    f = (k + 1) // 2
    c = (2 * f - 1 - f % 2) / (2 * f)
    return [1.0 - abs(x / f - c) for x in range(k)]


def up_matrix(n, s, device="cpu"):
    """[s n, n] float64 M of the bilinear conv2d_transpose with kernel 2s, stride s, SAME (pad s/2) along one axis:
    out[o] = sum_i M[o, i] in[i], M[o, i] = W[o - s i + s/2].  Its transpose is the adjoint."""
    k, pad = 2 * s, s // 2
    taps = torch.tensor(bilinear_taps(k), dtype=torch.float64)
    t = torch.arange(s * n)[:, None] - s * torch.arange(n)[None, :] + pad
    ok = (t >= 0) & (t < k)
    return torch.where(ok, taps[t.clamp(0, k - 1)], torch.zeros(())).to(device)


def up(x, s):
    """Bilinear x s up-sampling of an NHWC tensor in float64, separably: rows, then columns."""
    x = x.double()
    My, Mx = up_matrix(x.shape[1], s, x.device), up_matrix(x.shape[2], s, x.device)
    return torch.einsum("xj,nyjc->nyxc", Mx, torch.einsum("yi,nijc->nyjc", My, x))


def down(d, s):
    """Adjoint of `up`: [B, s h, s w, C] -> [B, h, w, C] in float64."""
    d = d.double()
    My, Mx = up_matrix(d.shape[1] // s, s, d.device), up_matrix(d.shape[2] // s, s, d.device)
    return torch.einsum("xj,nixc->nijc", Mx, torch.einsum("yi,nyxc->nixc", My, d))


def first_argmax(s):
    """Index of the first maximum over the last axis (tf.argmax; the kernels' lowest-index-wins rule)."""
    C = s.shape[-1]
    idx = torch.arange(C, device=s.device).expand_as(s)
    return torch.where(s == s.amax(-1, keepdim=True), idx, torch.full_like(idx, C)).amin(-1)


def f32(x):
    return np.float32(x)


# ---------------------------------------------------------------------------------------------------------------------
# add = a4 + up2(a5) and its adjoint (k_add_up2 / k_up2_bwd), the 1/8-resolution pack (k_pack_lowres), the 1x1 heads
# (k_lowres_heads)
# ---------------------------------------------------------------------------------------------------------------------
def add_up2(a4, a5, unit):
    """a4 + up2(a5) with operands on the grid `unit`; the terms are multiples of unit / 16.  Returns (add, budget)."""
    check_grid("a4", a4, unit)
    check_grid("a5", a5, unit)
    out = a4.double() + up(a5, 2)
    budget = check_budget("add_up2", (a4.double().abs() + up(a5.abs(), 2)).max() / (unit / 16))
    return out, budget


def up2_bwd(dadd, y5, unit):
    """d a5 = [y5 > 0] * up2^T(d add) (no mask when y5 is None), dadd on the grid `unit`.  Returns (d5, budget)."""
    check_grid("dadd", dadd, unit)
    d5 = down(dadd, 2)
    if y5 is not None:
        d5 = d5 * (y5.double() > 0)
    budget = check_budget("up2_bwd", down(dadd.abs(), 2).max() / (unit / 16))
    return d5, budget


def pack_lowres(sc, vt, C):
    """[score part: first C channels of sc | vertex part: first 3C channels of vt] as float64."""
    return torch.cat([sc[..., :C].double(), vt[..., :3 * C].double()], 3)


def lowres_heads(s4, s5, v4, v5, Ws, Wv, C, unit_x, unit_w):
    """k_lowres_heads: add = branch4 + up2(branch5) for both heads, then the two 1x1 matrices (Ws [Cs][C], Wv [Cv][3C]).
    Folded (Wv is None): the vertex outputs are add_v's first 3C channels.  Activations on the grid unit_x, weights on
    unit_w.  Returns ([B,h,w,4C], budget)."""
    add_s, b1 = add_up2(s4, s5, unit_x)
    add_v, b2 = add_up2(v4, v5, unit_x)
    check_grid("Ws", Ws, unit_w)
    g = unit_x / 16 * unit_w
    sc = add_s @ Ws.double()
    b3 = check_budget("lowres_heads score", (add_s.abs() @ Ws.double().abs()).max() / g)
    if Wv is None:
        return torch.cat([sc, add_v[..., :3 * C]], 3), max(b1, b2, b3)
    check_grid("Wv", Wv, unit_w)
    vt = add_v @ Wv.double()
    b4 = check_budget("lowres_heads vertex", (add_v.abs() @ Wv.double().abs()).max() / g)
    return torch.cat([sc, vt], 3), max(b1, b2, b3, b4)


# ---------------------------------------------------------------------------------------------------------------------
# up8 heads (k_up8_heads / k_up8_label): bilinear x8 + bias, ReLU, first-index arg-max, softmax
# ---------------------------------------------------------------------------------------------------------------------
def up8_heads(lowres, bias_s, bias_v, C, unit):
    """Dense heads from the 1/8-resolution tensor [B,h,w,4C] (lowres and biases on the grid `unit`; the terms are multiples
    of unit / 256).  Returns dict(score, vertex, label, prob, budget); prob is the float64 softmax of the exact scores."""
    check_grid("lowres", lowres, unit)
    check_grid("bias_s", bias_s, unit)
    check_grid("bias_v", bias_v, unit)
    bias = torch.cat([bias_s, bias_v]).double()
    u = up(lowres, 8)
    budget = check_budget("up8_heads", (up(lowres.abs(), 8) + bias.abs()).max() / (unit / 256))
    u = u + bias
    score = u[..., :C].clamp(min=0)
    return dict(score=score, vertex=u[..., C:], label=first_argmax(score), prob=torch.softmax(score, -1), budget=budget)


def softmax_bound(prob_ref, C):
    """|prob - prob_ref| bound of k_up8_heads' fp32 softmax: exp(s - max) with s - max exact, each expf within 2 ulp
    (relative 2^-22), the sum of C terms in C - 1 sequential fp32 additions (gamma_(C-1), u = 2^-24 each), the quotient
    rounded once (u).  Relative bound on numerator, denominator and quotient, with a 1e-6 margin for second-order terms."""
    u = 2.0 ** -24
    rel = (2.0 ** -22 + (2.0 ** -22 + (C - 1) * u / (1 - (C - 1) * u)) + u) * (1 + 1e-6)
    return rel * prob_ref


# ---------------------------------------------------------------------------------------------------------------------
# The up-sampling adjoint of both losses (k_up8_bwd_strip): d lowres from d up formed per pixel
# ---------------------------------------------------------------------------------------------------------------------
def coord_scale(extents):
    """coord_scale (csrc/heads_common.cuh) in float32: a = 1 / span, b = -vmin / span (0, 0 where span <= 0).  [C,3,2]."""
    e = extents.cpu().numpy().astype(np.float32)
    vmin, vmax = -e / f32(2), e / f32(2)
    span = vmax - vmin
    ok = span > 0
    a = np.where(ok, f32(1) / np.where(ok, span, f32(1)), f32(0)).astype(np.float32)
    b = np.where(ok, (f32(-1) * vmin) / np.where(ok, span, f32(1)), f32(0)).astype(np.float32)
    return torch.from_numpy(np.stack([a, b], -1))


def up8_bwd(P, sigma, thr, pv_unit, prob_unit=0.125):
    """Reference of pcnn_up8_heads_bwd with the 2-D (P["coord"] False) or the 3-D target (True) on problem P
    (up8_bwd_problem).  pv_unit: grid of the predicted vertex values and (2-D log z / 3-D) targets.

    d up, score channel c: s_cls * sel_p * (prob[p, c] - [c == gt_p]) * [score[p, c] > 0], s_cls = up_cls / (count + 1e-10f),
    sel_p = 0 <= gt_p < C and (gt_p > 0 or prob[p, 0] < thr).  Vertex channel 3g + k at pixels labelled 0 < g < C with a listed
    centre: s_vtx * w * dt, dt = smooth-L1'(w (pred - target)) (diff sigma^2 inside 1 / sigma^2, its sign outside).
    d lowres = up8^T(d up) per image; d bias = sum of d up over every pixel.

    Budgets: the per-output sums of |terms| (in units of d up's granularity / 256) and the bias sums over all pixels of the
    batch (in units of d up's granularity).  A vertical partial sum of the kernel is a sub-sum of its output's terms on a
    16x coarser grid, and every horizontal tap is >= 1/16, so the output budget bounds it too."""
    B, h, w, C = P["B"], P["h"], P["w"], P["C"]
    H, W = 8 * h, 8 * w
    dev = P["prob"].device
    s2 = f32(sigma) * f32(sigma)
    s_cls = f32(P["up_cls"]) / (f32(P["count"]) + f32(1e-10))
    s_vtx = f32(P["up_vtx"]) / (f32(P["sumw"]) + f32(1e-10))
    wi = float(P["w_inside"])
    for name, v in (("s_cls", s_cls), ("s_vtx", s_vtx), ("sigma^2", s2), ("w_inside", wi)):
        assert math.frexp(float(v))[0] == 0.5, f"{name} = {v} is not a power of two"
    s_cls, s_vtx, s2 = float(s_cls), float(s_vtx), float(s2)
    unit_s = s_cls * prob_unit
    unit_v = s_vtx * wi * min(1.0, wi * s2 * pv_unit)
    check_grid("prob", P["prob"], prob_unit)
    coord = P["coord"]
    if coord:
        ab = coord_scale(P["extents"]).double().to(dev)                          # [C,3,2]
    d_sc, d_vt = [], []
    bias_abs = torch.zeros(4 * C, dtype=torch.float64, device=dev)
    bias = torch.zeros(4 * C, dtype=torch.float64, device=dev)
    budget = 0.0
    for n in range(B):
        gt = P["gt"][n].long()
        valid = (gt >= 0) & (gt < C)
        g0 = torch.where(valid, gt, torch.zeros_like(gt))
        prob = P["prob"][n].double()
        sel = valid & ((gt > 0) | (prob[..., 0] < thr))
        onehot = torch.nn.functional.one_hot(g0, C).double()
        ds = s_cls * sel[..., None] * (prob - onehot) * (P["score"][n] > 0)
        # vertex part
        listed = valid & (gt > 0) & (P["centers"][n, g0, 2] > 0)
        pv = P["pv"][n].double().view(H, W, C, 3).gather(2, g0[..., None, None].expand(H, W, 1, 3))[:, :, 0]   # [H,W,3]
        if coord:
            v = P["vertmap"][n].double()
            a, b = ab[g0, :, 0], ab[g0, :, 1]
            tg = (a * v).float().double() + b                                    # a v rounded, then + b (exact on the grids used)
            assert bool((tg.float().double() == tg).all()), "3-D targets must be exact in fp32"
            fine = torch.ones(3, dtype=torch.bool, device=dev)
        else:
            cen = P["centers"][n, g0]                                            # [H,W,3]
            ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
            dx, dy = cen[..., 0].double() - xs, cen[..., 1].double() - ys
            nrm = (dx * dx + dy * dy).sqrt() + 1e-10
            lz = torch.where(cen[..., 2] > 0, cen[..., 2].double().clamp(min=1e-30).log(), torch.zeros((), dtype=torch.float64, device=dev))
            tg = torch.stack([(dx / nrm).float().double(), (dy / nrm).float().double(), lz.float().double()], -1)
            # direction channels stay in the linear regime: |pred| >= 1 + 1 / (sigma^2 w) >= |target| + 1 / (sigma^2 w), and fp32
            # rounding is monotone, so the kernel's |w (pred - target)| >= 1 / sigma^2 as well; only the sign enters d up
            far = pv[..., :2].abs() >= 1.0 + 1.0 / (s2 * wi)
            assert bool((far | ~listed[..., None]).all()), "a direction channel left the linear regime"
            fine = torch.tensor([False, False, True], device=dev)
        diff = wi * (pv - tg)
        quad = diff.abs() < 1.0 / s2
        dt = torch.where(quad, diff * s2, diff.sign())
        m = listed[..., None] & fine
        check_grid("vertex pred - target", torch.where(m, pv - tg, torch.zeros((), dtype=torch.float64, device=dev)), pv_unit)
        dv_own = s_vtx * wi * dt * listed[..., None]
        dv = torch.zeros(H, W, C, 3, dtype=torch.float64, device=dev)
        dv.scatter_(2, g0[..., None, None].expand(H, W, 1, 3), dv_own[:, :, None, :])
        dv = dv.view(H, W, 3 * C)
        check_grid("d up (score)", ds, unit_s)
        check_grid("d up (vertex)", dv, unit_v)
        d_up = torch.cat([ds, dv], 2)[None]
        units = torch.cat([torch.full((C,), unit_s), torch.full((3 * C,), unit_v)]).to(dev).double()
        out = down(d_up, 8)[0]
        budget = max(budget, check_budget("up8_bwd output", (down(d_up.abs(), 8)[0] / (units / 256)).max()))
        d_sc.append(out[..., :C])
        d_vt.append(out[..., C:])
        bias += d_up[0].sum((0, 1))
        bias_abs += d_up[0].abs().sum((0, 1))
        del d_up
    budget = max(budget, check_budget("up8_bwd bias", (bias_abs / torch.cat([torch.full((C,), unit_s), torch.full((3 * C,), unit_v)])
                                                                 .to(dev).double()).max()))
    return dict(d_sc=torch.stack(d_sc), d_vt=torch.stack(d_vt), dbias=bias, budget=budget)


def up8_bwd_problem(B, h, w, C, coord, gen, device="cpu", w_inside=4.0, up_cls=1.0, up_vtx=2.0, count=1024.0, sumw=1024.0):
    """Operands of the up-sampling adjoint on dyadic grids.

    prob: multiples of 1/8 in [0, 1] (the kernel reads prob and score as given: no softmax needed), so background pixels have
    prob[.., 0] below, at and above a threshold of 1/2, and at and below 1.  score: ReLU of multiples of 1/8, a third exactly 0.
    gt: -1, values >= C and < -1, background 0 and foreground classes; image 0 lists every class but 2, image 1 the odd ones
    (none at C = 2).  Normalisers count = sum w = 1024: the scales up / (n + 1e-10f) are powers of two.
    Vertex head: the 1/8-resolution vertex channels are multiples of 1/4, biases multiples of 1/8, so the predictions lie on a
    2^-10 grid.  2-D: the two direction channels keep |pred| >= 1 + 1 / w_inside (linear regime for sigma >= 1) through a signed
    bias, listed centres have z = 1, so the log-z target is 0 and the third channel crosses into the quadratic regime.  3-D:
    extents 0.25, 0.5, 1 (a = 4, 2, 1, b = 1/2), a zero-extent axis for class 1, vertmap on a 1/256 grid.
    Foreground is 45 % of the pixels (15 % at C = 2, where one class takes all of it) so that each class's vertex-bias sum
    stays inside the budget."""
    H, W = 8 * h, 8 * w
    lowres = dyadic((B, h, w, 4 * C), -1, 1, 0.25, gen)
    bias_v = dyadic((3 * C,), -0.25, 0.25, 0.125, gen)
    if coord:
        lowres[..., C:] = dyadic((B, h, w, 3 * C), -0.5, 0.5, 0.25, gen)
        bias_v[:] = 0.5
    else:
        sign = torch.where(int_operands((C, 2), 0, 1, gen) > 0, 1.0, -1.0)
        lv = lowres[..., C:].view(B, h, w, C, 3)
        lv[..., :2] = sign * dyadic((B, h, w, C, 2), 0, 1, 0.25, gen)
        bv = bias_v.view(C, 3)
        bv[:, :2] = sign * (1.0 + 1.0 / w_inside + dyadic((C, 2), 0, 0.5, 0.125, gen))
    prob = dyadic((B, H, W, C), 0, 1, 0.125, gen)
    score = dyadic((B, H, W, C), -1, 2, 0.125, gen).clamp(min=0)
    r = int_operands((B, H, W), 0, 99, gen).long()
    fg_pct = 45 if C > 2 else 15
    fg = 1 + int_operands((B, H, W), 0, C - 2, gen).long() if C > 2 else torch.ones((B, H, W), dtype=torch.long)
    gt = torch.where(r < 8, -1, torch.where(r < 10, C + r, torch.where(r < 12, -2 - r, torch.where(r < 100 - fg_pct, 0, fg))))
    centers = torch.zeros(B, C, 3)
    centers[:, :, 0] = dyadic((B, C), 0, W, 0.5, gen)
    centers[:, :, 1] = dyadic((B, C), 0, H, 0.5, gen)
    centers[0, 1:, 2] = 1.0
    if C > 2:
        centers[0, 2, 2] = 0.0                                                  # class 2: labelled but not listed
    if B > 1 and C > 2:
        centers[1, 1::2, 2] = 1.0
    P = dict(B=B, h=h, w=w, C=C, coord=coord, lowres=lowres, bias_v=bias_v, prob=prob, score=score, gt=gt.to(torch.int32),
             centers=centers, w_inside=w_inside, up_cls=up_cls, up_vtx=up_vtx, count=count, sumw=sumw)
    if coord:
        ext = torch.tensor([0.25, 0.5, 1.0])[(torch.arange(C)[:, None] + torch.arange(3)[None, :]) % 3]
        ext[1, 2] = 0.0                                                          # a zero-extent axis: a = b = 0, target 0
        P["extents"] = ext.contiguous()
        P["vertmap"] = dyadic((B, H, W, 3), -0.5, 0.5, 1.0 / 256, gen)
    P = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in P.items()}
    # the dense vertex prediction up8(lowres) + bias, exact on the 2^-10 grid (its budget is checked here)
    P["pv"] = up8_heads(P["lowres"], torch.zeros(C, device=device), P["bias_v"], C, 0.125)["vertex"]
    return P


def run_up8_bwd(P, sigma, thr, Cv):
    """The adjoint (posecnn_b200.heads.up8_heads_bwd) on problem P on the GPU, into outputs pre-filled with 7 so that padding
    channels must be written as 0; d_vt has channel stride Cv.  Returns (d_sc, d_vt, dbias)."""
    from posecnn_b200 import heads
    B, h, w, C = P["B"], P["h"], P["w"], P["C"]
    dev = P["prob"].device
    out = (torch.full((B, h, w, 64), 7.0, dtype=torch.bfloat16, device=dev), torch.full((B, h, w, Cv), 7.0, dtype=torch.bfloat16, device=dev),
           torch.full((4 * C,), 7.0, device=dev))
    cls_out = torch.tensor([0.5, P["count"]], device=dev)
    vtx_out = torch.tensor([0.25, P["sumw"]], device=dev)
    vm, ext = (P["vertmap"], P["extents"]) if P["coord"] else (None, None)
    return heads.up8_heads_bwd(P["prob"], P["score"], P["gt"], cls_out, P["up_cls"], thr, P["lowres"], P["bias_v"], P["centers"], vtx_out,
                               P["up_vtx"], P["w_inside"], sigma, vertmap=vm, extents=ext, out=out)


# ---------------------------------------------------------------------------------------------------------------------
# The classification loss of the training step (k_loss_cls_hard_raw): Hardlabel-selected cross entropy from raw scores
# ---------------------------------------------------------------------------------------------------------------------
def ulp32(x):
    """Spacing of fp32 numbers at |x| (2^-149 at 0)."""
    x = x.abs().double().clamp(min=2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(x)) - 23)


def loss_cls_hard_raw(score_raw, prob, gt, thr):
    """-mean over selected pixels of log_softmax(score_raw)[gt] in float64, with the count and an error bound for the kernel.

    Per selected pixel the kernel forms t = (s_g - m) - logf(sum_c expf(s_c - m)) in fp32 with s - m exact (dyadic scores):
    each expf within 2 ulp (2^-22 relative), C - 1 sequential additions (gamma_(C-1)), so the sum is within r_C = 2^-22 +
    gamma_(C-1) relative and its log within r_C absolute (with a 1e-6 margin); logf adds 1 ulp of its result and the final
    subtraction half an ulp of t.  The double accumulation is taken as exact; the quotient and its fp32 store add 2^-23
    relative.  Returns (loss, count, bound, logsm) with logsm the float64 log-softmax [..., C]."""
    C = score_raw.shape[-1]
    s = score_raw.double()
    m = s.amax(-1, keepdim=True)
    lse = (s - m).exp().sum(-1)
    logsm = s - m - lse.log()[..., None]
    gtl = gt.long()
    valid = (gtl >= 0) & (gtl < C)
    g0 = torch.where(valid, gtl, torch.zeros_like(gtl))
    sel = valid & ((gtl > 0) | (prob.double()[..., 0] < thr))
    t = logsm.gather(-1, g0[..., None])[..., 0]
    n = int(sel.sum())
    loss = float(-(t * sel).sum() / (n + 1e-10))
    u = 2.0 ** -24
    r_c = (2.0 ** -22 + (C - 1) * u / (1 - (C - 1) * u)) * (1 + 1e-6)
    per = r_c + 2 * ulp32(lse.log()) + ulp32(t)           # ulps counted one binade up: the fp32 values may cross a power of two
    bound = float((per * sel).sum() / max(n, 1)) + 2.0 ** -23 * abs(loss)
    return loss, n, bound, logsm


# ---------------------------------------------------------------------------------------------------------------------
# Launch plans: the grid / loop formulas of the entry points, so that each test states (and asserts) what it covered
# ---------------------------------------------------------------------------------------------------------------------
def vertex_stride(C):
    """Channel stride Cv of the vertex-head tensors for C classes: the network's 128, or where 3C > 128 (C = 50) the next
    multiple of 32 (the entry points require Cv >= 3C)."""
    return max(128, -(-3 * C // 32) * 32)


def ew_plan(total):
    """Grid-stride kernels of csrc/train_bwd.cu (ew_blocks): min(ceil(total / 256), kNumSMs * 8) blocks of 256 threads."""
    blocks = min((total + 255) // 256, NUM_SMS * 8)
    return dict(total=total, blocks=blocks, iters=-(-total // (blocks * 256)))


def ew_batch_for_coverage(per_image, iters=2):
    """Smallest batch whose grid-stride loop runs at least `iters` iterations; returns (B, plan)."""
    B = 1
    while ew_plan(B * per_image)["iters"] < iters:
        B += 1
    return B, ew_plan(B * per_image)


def lowres_heads_plan(B, h, w, C, Cs=64, Cv=128, folded=False):
    """pcnn_lowres_heads: warps of 8-pixel groups (block cap kNumSMs x 2, folded x 8) and the column map of phase 2."""
    npix = B * h * w
    groups = -(-npix // 8)
    blocks = min(-(-npix // 64), NUM_SMS * (8 if folded else 2))
    warps = 8 * blocks
    C3 = 0 if folded else 3 * C
    split = Cv // Cs
    n_full, v_left = C3 // 32, C3 - 32 * (C3 // 32)
    tail_start = -(-C // split) * split
    tail = -(-(tail_start + v_left * split) // 32)
    return dict(npix=npix, groups=groups, blocks=blocks, warps=warps, groups_per_warp=-(-groups // warps),
                ragged_group=npix % 8 != 0, full_passes=n_full, tail_passes=tail, split_columns=v_left)


def up8_heads_plan(B, h, w, C, label_only=False):
    """pcnn_up8_heads: the label-only kernel k_up8_label when its 11 w C floats fit 200 KB, else k_up8_heads on 20-cell
    segments."""
    smem_l = 4 * 11 * w * C
    if label_only and smem_l <= 200 * 1024:
        return dict(kernel="k_up8_label", grid=(h, B), smem=smem_l)
    seg = min(w, 20)
    return dict(kernel="k_up8_heads", grid=(8 * h, B, -(-w // seg)), segments=-(-w // seg), ragged_segment=w % seg != 0,
                smem=4 * ((seg + 2) * 4 * C + 8 * seg * C + 16 * seg))


def up8_bwd_plan(B, h, w, C):
    """pcnn_up8_heads_bwd: CTAs of strips (4 cells, 16 at C = 2) x bands of 16 low-resolution rows x images,
    (8 SC + 8) C / 2 threads, instantiation <22>, <2> or the generic <0>; 4C partial bias floats per CTA.  smem is the 2-D
    mode's (the 3-D mode adds 6C floats)."""
    sc = 16 if C == 2 else 4
    strips, bands = -(-w // sc), -(-h // 16)
    return dict(kernel="<%d>" % (C if C in (2, 22) else 0), strip=sc, strips=strips, bands=bands, ctas=B * strips * bands,
                threads=(8 * sc + 8) * (C // 2), last_strip_cells=w - sc * (strips - 1), last_band_rows=h - 16 * (bands - 1),
                smem=4 * ((8 * sc + 8) * 11 * C + C), workspace=4 * B * strips * bands * 4 * C)
